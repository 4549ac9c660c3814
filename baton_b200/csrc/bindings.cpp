// PyTorch bindings for the sm_90a kernels.  Thin by design: shape logic lives in Python
// (baton_b200/ops), this file only unwraps tensors, picks the current stream and checks codes.
#include <ATen/cuda/CUDAContext.h>
#include <c10/cuda/CUDAGuard.h>
#include <torch/extension.h>

#include <optional>
#include <vector>

#include "launch.h"

namespace {

inline cudaStream_t cur_stream() { return at::cuda::getCurrentCUDAStream().stream(); }
inline void check(int rc, const char* what) {
  TORCH_CHECK(rc == 0, "baton_b200::", what, " failed with code ", rc,
              rc > 0 ? std::string(" (") + cudaGetErrorString(static_cast<cudaError_t>(rc)) + ")" : std::string());
}
inline const void* cptr(const at::Tensor& t) { return t.data_ptr(); }
inline void* ptr(at::Tensor& t) { return t.data_ptr(); }
template <class T>
inline T* opt_ptr(const std::optional<at::Tensor>& t) {
  return (t.has_value() && t->defined()) ? reinterpret_cast<T*>(t->data_ptr()) : nullptr;
}
#define CHECK_CUDA(x) TORCH_CHECK((x).is_cuda(), #x " must be a CUDA tensor")

// FedProx anchor of an SGD step: fp32, contiguous, at least as long as the parameters it anchors, with a 5-float hyper
inline const float* prox_anchor(const std::optional<at::Tensor>& anchor, int64_t numel, const at::Tensor& hyper) {
  if (!anchor.has_value() || !anchor->defined()) return nullptr;
  CHECK_CUDA(*anchor);
  TORCH_CHECK(anchor->scalar_type() == at::kFloat && anchor->is_contiguous() && anchor->numel() >= numel,
              "prox anchor: contiguous fp32 covering the parameters");
  TORCH_CHECK(hyper.numel() >= 5, "prox anchor: hyper needs 5 floats {lr, momentum, weight_decay, dampening, prox_mu}");
  return anchor->data_ptr<float>();
}

// SCAFFOLD correction of an SGD step: fp32, contiguous, at least as long as the parameters it corrects; no anchor
inline const float* scaf_corr(const std::optional<at::Tensor>& corr, int64_t numel, const float* anchor) {
  if (!corr.has_value() || !corr->defined()) return nullptr;
  CHECK_CUDA(*corr);
  TORCH_CHECK(corr->scalar_type() == at::kFloat && corr->is_contiguous() && corr->numel() >= numel,
              "scaffold correction: contiguous fp32 covering the parameters");
  TORCH_CHECK(anchor == nullptr, "an SGD step takes a FedProx anchor or a SCAFFOLD correction, not both");
  return corr->data_ptr<float>();
}

// AdamW second moment of an optimizer step: fp32, contiguous, at least as long as the parameters; it needs the first
// moment (the momentum buffer), the step's AdamW row as `hyper` (ADAMW_ROW = 12 floats) and no FedProx / SCAFFOLD term
inline float* adam_v_ptr(const std::optional<at::Tensor>& v, int64_t numel, const float* mom, const at::Tensor& hyper,
                         const float* anchor, const float* corr) {
  if (!v.has_value() || !v->defined()) return nullptr;
  CHECK_CUDA(*v);
  TORCH_CHECK(v->scalar_type() == at::kFloat && v->is_contiguous() && v->numel() >= numel,
              "adamw second moment: contiguous fp32 covering the parameters");
  TORCH_CHECK(mom != nullptr, "an AdamW step needs the first-moment (momentum) buffer");
  TORCH_CHECK(hyper.numel() >= 12, "an AdamW step takes its step row (12 floats) as hyper");
  TORCH_CHECK(anchor == nullptr && corr == nullptr, "an AdamW step takes no FedProx anchor or SCAFFOLD correction");
  return v->data_ptr<float>();
}

// optimizer epilogue of a weight-gradient GEMM: theta / theta_bf16 / momentum / anchor / correction / second moment
// start at the element of D[0, 0]
inline std::optional<B200SgdEpilogue> sgd_epilogue(const std::optional<at::Tensor>& theta,
                                                   const std::optional<at::Tensor>& theta_bf16,
                                                   const std::optional<at::Tensor>& mom,
                                                   const std::optional<at::Tensor>& hyper, bool nesterov,
                                                   const std::optional<at::Tensor>& anchor,
                                                   const std::optional<at::Tensor>& corr,
                                                   const std::optional<at::Tensor>& adam_v) {
  if (!hyper.has_value() || !hyper->defined()) return std::nullopt;
  TORCH_CHECK(theta.has_value() && theta->scalar_type() == at::kFloat && hyper->scalar_type() == at::kFloat &&
                  (!theta_bf16.has_value() || theta_bf16->scalar_type() == at::kBFloat16) &&
                  (!mom.has_value() || mom->scalar_type() == at::kFloat),
              "sgd epilogue: fp32 theta / momentum / hyper, bf16 shadow");
  const float* a = prox_anchor(anchor, theta->numel(), *hyper);
  // theta runs to the end of the arena, the correction to the end of the parameters: the GEMM only addresses its
  // output's elements, which are parameters
  const float* c = scaf_corr(corr, 0, a);
  return B200SgdEpilogue{theta->data_ptr<float>(), opt_ptr<void>(theta_bf16), opt_ptr<float>(mom),
                         hyper->data_ptr<float>(), nesterov ? 1 : 0, a, c,
                         adam_v_ptr(adam_v, 0, opt_ptr<float>(mom), *hyper, a, c)};
}

// eval-mode BatchNorm epilogue of a forward GEMM: fp32 [N] scale and shift, optional bf16 residual rows
inline std::optional<B200AffineEpilogue> affine_epilogue(const std::optional<at::Tensor>& scale,
                                                         const std::optional<at::Tensor>& shift,
                                                         const std::optional<at::Tensor>& residual, bool relu,
                                                         int64_t rows, int64_t N) {
  if (!scale.has_value() || !scale->defined()) return std::nullopt;
  TORCH_CHECK(shift.has_value() && shift->defined(), "affine epilogue: scale without shift");
  CHECK_CUDA(*scale); CHECK_CUDA(*shift);
  TORCH_CHECK(scale->scalar_type() == at::kFloat && shift->scalar_type() == at::kFloat &&
                  scale->is_contiguous() && shift->is_contiguous() && scale->numel() >= N && shift->numel() >= N,
              "affine epilogue: fp32 [N] scale / shift");
  long long ldr = 0;
  if (residual.has_value() && residual->defined()) {
    CHECK_CUDA(*residual);
    TORCH_CHECK(residual->scalar_type() == at::kBFloat16 && residual->stride(-1) == 1 && residual->size(-1) == N &&
                    residual->numel() >= rows * N,
                "affine epilogue: bf16 [rows, N] residual with unit inner stride");
    ldr = residual->dim() >= 2 ? residual->stride(-2) : N;
  }
  return B200AffineEpilogue{scale->data_ptr<float>(), shift->data_ptr<float>(), opt_ptr<const void>(residual), ldr,
                            relu ? 1 : 0};
}

// ---- in-graph kernel timeline (pdl.cuh): every translation unit owns a copy of the trace pointer
extern "C" {
#define B200_TRACE_TUS(X) X(gemm_wgmma) X(gemm_fp8) X(quant) X(attention) X(im2col_tma) X(gemm_simt) X(fedavg) \
  X(elementwise) X(conv) X(norm) X(loss) X(conv_halo)
#define B200_DECL(tu) int b200_trace_set_##tu(unsigned long long* p);
B200_TRACE_TUS(B200_DECL)
#undef B200_DECL
}
// buf: int64 CUDA tensor [2 + 2 * capacity] ({cursor, capacity, (t_ns, tag)...}) or None to stop tracing.
// Returns false when the extension was not built with -DB200_TRACE.
bool trace_set(const std::optional<at::Tensor>& buf) {
  unsigned long long* p = nullptr;
  if (buf.has_value() && buf->defined()) {
    CHECK_CUDA(*buf);
    TORCH_CHECK(buf->scalar_type() == at::kLong && buf->is_contiguous() && buf->numel() >= 4, "trace buffer: int64 [2+2n]");
    p = reinterpret_cast<unsigned long long*>(buf->data_ptr());
  }
  int rc = 0;
#define B200_SET(tu) rc |= b200_trace_set_##tu(p);
  B200_TRACE_TUS(B200_SET)
#undef B200_SET
  return rc == 0;
}

// false: the optimizer or BatchNorm epilogue was requested and declined (nothing was written)
bool gemm(const at::Tensor& a, const at::Tensor& b, at::Tensor d, const std::optional<at::Tensor>& bias, int64_t M,
          int64_t N, int64_t K, int64_t lda, int64_t ldb, int64_t ldd, bool a_mn, bool b_mn, int64_t act,
          int64_t split_k, bool accumulate, double alpha, const std::optional<at::Tensor>& flags, int64_t flag_epoch,
          int64_t flag_elem_off, int64_t flag_tile_elems, int64_t flag_bias_off, int64_t force_bn, bool simt,
          const std::optional<at::Tensor>& col_stats, const std::optional<at::Tensor>& flag_epoch_word,
          const std::optional<at::Tensor>& sgd_theta, const std::optional<at::Tensor>& sgd_theta_bf16,
          const std::optional<at::Tensor>& sgd_mom, const std::optional<at::Tensor>& sgd_hyper, bool sgd_nesterov,
          const std::optional<at::Tensor>& sgd_anchor, const std::optional<at::Tensor>& sgd_corr,
          const std::optional<at::Tensor>& sgd_v, const std::optional<at::Tensor>& bn_scale, const std::optional<at::Tensor>& bn_shift,
          const std::optional<at::Tensor>& residual, bool bn_relu) {
  CHECK_CUDA(a); CHECK_CUDA(b); CHECK_CUDA(d);
  TORCH_CHECK(a.scalar_type() == at::kBFloat16 && b.scalar_type() == at::kBFloat16, "gemm operands must be bf16");
  TORCH_CHECK(d.scalar_type() == at::kBFloat16 || d.scalar_type() == at::kFloat, "gemm output must be bf16/fp32");
  const c10::cuda::CUDAGuard guard(a.device());
  const int out_fp32 = d.scalar_type() == at::kFloat;
  const float* bp = opt_ptr<const float>(bias);
  TORCH_CHECK(!col_stats.has_value() || (!simt && col_stats->scalar_type() == at::kFloat && col_stats->numel() >= 2 * N),
              "col_stats needs the tensor-core path and a [2N] fp32 buffer");
  if (simt) {
    TORCH_CHECK(!sgd_hyper.has_value(), "the SIMT GEMM has no optimizer epilogue");
    TORCH_CHECK(!bn_scale.has_value(), "the SIMT GEMM has no BatchNorm epilogue");
    check(b200_gemm_simt(cptr(a), cptr(b), ptr(d), bp, M, N, K, lda, ldb, ldd, a_mn, b_mn, out_fp32, act, accumulate,
                         static_cast<float>(alpha), cur_stream()),
          "gemm_simt");
    return true;
  }
  const std::optional<B200SgdEpilogue> sgd =
      sgd_epilogue(sgd_theta, sgd_theta_bf16, sgd_mom, sgd_hyper, sgd_nesterov, sgd_anchor, sgd_corr, sgd_v);
  const std::optional<B200AffineEpilogue> affine = affine_epilogue(bn_scale, bn_shift, residual, bn_relu, M, N);
  const int rc = b200_gemm_bf16(cptr(a), cptr(b), ptr(d), bp, M, N, K, lda, ldb, ldd, a_mn, b_mn, out_fp32, act, split_k,
                                accumulate, static_cast<float>(alpha), opt_ptr<const uint32_t>(flags),
                                static_cast<uint32_t>(flag_epoch), flag_elem_off, static_cast<int>(flag_tile_elems),
                                flag_bias_off, static_cast<int>(force_bn), opt_ptr<float>(col_stats),
                                opt_ptr<const uint32_t>(flag_epoch_word), sgd ? &*sgd : nullptr,
                                affine ? &*affine : nullptr, cur_stream());
  if (rc == B200_SGD_EPILOGUE_DECLINED || rc == B200_AFFINE_EPILOGUE_DECLINED) return false;
  check(rc, "gemm_bf16");
  return true;
}

void gemm_batched(const at::Tensor& a, const at::Tensor& b, at::Tensor d, int64_t M, int64_t N, int64_t K, int64_t lda,
                  int64_t ldb, int64_t ldd, bool a_mn, bool b_mn, int64_t act, double alpha, int64_t n_outer,
                  int64_t n_inner, int64_t a_outer, int64_t a_inner, int64_t b_outer, int64_t b_inner, int64_t d_outer,
                  int64_t d_inner, bool accumulate) {
  CHECK_CUDA(a); CHECK_CUDA(b); CHECK_CUDA(d);
  TORCH_CHECK(a.scalar_type() == at::kBFloat16 && b.scalar_type() == at::kBFloat16, "gemm operands must be bf16");
  const c10::cuda::CUDAGuard guard(a.device());
  check(b200_gemm_bf16_batched(cptr(a), cptr(b), ptr(d), M, N, K, lda, ldb, ldd, a_mn, b_mn,
                               d.scalar_type() == at::kFloat, act, static_cast<float>(alpha), n_outer, n_inner, a_outer,
                               a_inner, b_outer, b_inner, d_outer, d_inner, accumulate, cur_stream()),
        "gemm_bf16_batched");
}

// fused attention forward (S = 128, d_head = 64); returns false when the shape is unsupported
bool attention_fwd(const at::Tensor& qkv, at::Tensor out, at::Tensor probs, int64_t B, int64_t S, int64_t H, int64_t dh,
                   double scale) {
  CHECK_CUDA(qkv); CHECK_CUDA(out); CHECK_CUDA(probs);
  TORCH_CHECK(qkv.scalar_type() == at::kBFloat16 && out.scalar_type() == at::kBFloat16 &&
              probs.scalar_type() == at::kBFloat16 && qkv.is_contiguous() && out.is_contiguous() && probs.is_contiguous());
  const c10::cuda::CUDAGuard guard(qkv.device());
  const int rc = b200_attention_fwd(cptr(qkv), ptr(out), ptr(probs), static_cast<int>(B), static_cast<int>(S),
                                    static_cast<int>(H), static_cast<int>(dh), static_cast<float>(scale), cur_stream());
  if (rc == -2) return false;
  check(rc, "attention_fwd");
  return true;
}

// probe: explicit-im2col-layout dump of TMA im2col loads (semantics probe for the implicit-GEMM conv)
bool im2col_tma_probe(const at::Tensor& x, at::Tensor col, int64_t kh, int64_t kw, int64_t stride, int64_t pad,
                      int64_t ho, int64_t wo) {
  CHECK_CUDA(x); CHECK_CUDA(col);
  TORCH_CHECK(x.scalar_type() == at::kBFloat16 && col.scalar_type() == at::kBFloat16 && x.dim() == 4 && x.is_contiguous() &&
              col.is_contiguous());
  const c10::cuda::CUDAGuard guard(x.device());
  const int rc = b200_im2col_tma_probe(cptr(x), ptr(col), static_cast<int>(x.size(0)), static_cast<int>(x.size(1)),
                                       static_cast<int>(x.size(2)), static_cast<int>(x.size(3)), static_cast<int>(kh),
                                       static_cast<int>(kw), static_cast<int>(stride), static_cast<int>(pad),
                                       static_cast<int>(ho), static_cast<int>(wo), cur_stream());
  if (rc == -2) return false;
  check(rc, "im2col_tma_probe");
  return true;
}

bool attention_bwd(const at::Tensor& qkv, const at::Tensor& dout, const at::Tensor& probs, at::Tensor dqkv, int64_t B,
                   int64_t S, int64_t H, int64_t dh, double scale) {
  CHECK_CUDA(qkv); CHECK_CUDA(dout); CHECK_CUDA(probs); CHECK_CUDA(dqkv);
  TORCH_CHECK(qkv.scalar_type() == at::kBFloat16 && dout.scalar_type() == at::kBFloat16 &&
              probs.scalar_type() == at::kBFloat16 && dqkv.scalar_type() == at::kBFloat16 && qkv.is_contiguous() &&
              dout.is_contiguous() && probs.is_contiguous() && dqkv.is_contiguous());
  const c10::cuda::CUDAGuard guard(qkv.device());
  const int rc = b200_attention_bwd(cptr(qkv), cptr(dout), cptr(probs), ptr(dqkv), static_cast<int>(B), static_cast<int>(S),
                                    static_cast<int>(H), static_cast<int>(dh), static_cast<float>(scale), cur_stream());
  if (rc == -2) return false;
  check(rc, "attention_bwd");
  return true;
}

// implicit-GEMM convolution; false = shape not supported (caller falls back to im2col + GEMM)
bool conv_igemm_fwd(const at::Tensor& x, const at::Tensor& w, at::Tensor y, int64_t kh, int64_t kw, int64_t stride,
                    int64_t pad, int64_t ho, int64_t wo, int64_t cluster_k, int64_t force_bn,
                    const std::optional<at::Tensor>& col_stats, const std::optional<at::Tensor>& bn_scale,
                    const std::optional<at::Tensor>& bn_shift, const std::optional<at::Tensor>& residual, bool bn_relu) {
  CHECK_CUDA(x); CHECK_CUDA(w); CHECK_CUDA(y);
  TORCH_CHECK(x.scalar_type() == at::kBFloat16 && w.scalar_type() == at::kBFloat16 && y.scalar_type() == at::kBFloat16 &&
              x.dim() == 4 && x.is_contiguous() && w.is_contiguous() && y.is_contiguous());
  TORCH_CHECK(y.numel() == x.size(0) * ho * wo * w.size(0), "conv_igemm_fwd: y must hold [N*Ho*Wo, Cout] elements");
  const c10::cuda::CUDAGuard guard(x.device());
  const std::optional<B200AffineEpilogue> affine =
      affine_epilogue(bn_scale, bn_shift, residual, bn_relu, x.size(0) * ho * wo, w.size(0));
  const int rc = b200_conv_igemm_fwd(cptr(x), cptr(w), ptr(y), static_cast<int>(x.size(0)), static_cast<int>(x.size(1)),
                                     static_cast<int>(x.size(2)), static_cast<int>(x.size(3)), static_cast<int>(w.size(0)),
                                     static_cast<int>(kh), static_cast<int>(kw), static_cast<int>(stride),
                                     static_cast<int>(pad), static_cast<int>(ho), static_cast<int>(wo),
                                     static_cast<int>(cluster_k), static_cast<int>(force_bn), opt_ptr<float>(col_stats),
                                     affine ? &*affine : nullptr, cur_stream());
  if (rc == -2 || rc == B200_AFFINE_EPILOGUE_DECLINED) return false;
  check(rc, "conv_igemm_fwd");
  return true;
}
// dx [N, H, W, Cin] = implicit dgrad of a stride-1 convolution; dy [N, Ho, Wo, Cout], w [Cout, KH*KW*Cin]
bool conv_igemm_dgrad(const at::Tensor& dy, const at::Tensor& w, at::Tensor dx, int64_t kh, int64_t kw, int64_t pad,
                      int64_t cluster_k, int64_t force_bn) {
  CHECK_CUDA(dy); CHECK_CUDA(w); CHECK_CUDA(dx);
  TORCH_CHECK(dy.scalar_type() == at::kBFloat16 && w.scalar_type() == at::kBFloat16 && dx.scalar_type() == at::kBFloat16 &&
              dy.dim() == 4 && dx.dim() == 4 && dy.is_contiguous() && w.is_contiguous() && dx.is_contiguous());
  const c10::cuda::CUDAGuard guard(dy.device());
  const int rc = b200_conv_igemm_dgrad(cptr(dy), cptr(w), ptr(dx), static_cast<int>(dx.size(0)), static_cast<int>(dx.size(1)),
                                       static_cast<int>(dx.size(2)), static_cast<int>(dx.size(3)), static_cast<int>(dy.size(3)),
                                       static_cast<int>(kh), static_cast<int>(kw), static_cast<int>(pad),
                                       static_cast<int>(dy.size(1)), static_cast<int>(dy.size(2)),
                                       static_cast<int>(cluster_k), static_cast<int>(force_bn), cur_stream());
  if (rc == -2) return false;
  check(rc, "conv_igemm_dgrad");
  return true;
}
// halo-tiled 3x3 stride-1 convolution: src [N, H, W, 64] (x forward, dy dgrad), w [Cout, 9*Cin], out [N*H*W, Nout]
// (Nout = Cout forward, Cin dgrad); false = shape not supported by the kernel
bool conv_halo(const at::Tensor& src, const at::Tensor& w, at::Tensor out, bool dgrad, int64_t mc,
               const std::optional<at::Tensor>& col_stats) {
  CHECK_CUDA(src); CHECK_CUDA(w); CHECK_CUDA(out);
  TORCH_CHECK(src.scalar_type() == at::kBFloat16 && w.scalar_type() == at::kBFloat16 && out.scalar_type() == at::kBFloat16 &&
              src.dim() == 4 && src.size(3) == 64 && src.is_contiguous() && w.is_contiguous() && out.is_contiguous());
  const int64_t rows = src.size(0) * src.size(1) * src.size(2);
  TORCH_CHECK(rows > 0 && out.numel() % rows == 0, "conv_halo: out must hold [N*H*W, Nout] elements");
  const int64_t nout = out.numel() / rows;
  TORCH_CHECK(w.numel() == (dgrad ? 64 * 9 * nout : nout * 9 * 64), "conv_halo: w must be [Cout, 9*Cin]");
  TORCH_CHECK(dgrad ? !col_stats.has_value()
                    : (!col_stats.has_value() || (col_stats->scalar_type() == at::kFloat && col_stats->numel() >= 2 * nout)),
              "conv_halo: col_stats is a [2 Cout] fp32 buffer of the forward");
  const c10::cuda::CUDAGuard guard(src.device());
  const int rc = b200_conv_halo(cptr(src), cptr(w), ptr(out), static_cast<int>(src.size(0)), static_cast<int>(src.size(1)),
                                static_cast<int>(src.size(2)), static_cast<int>(nout), dgrad ? 1 : 0,
                                static_cast<int>(mc), opt_ptr<float>(col_stats), cur_stream());
  if (rc == -2) return false;
  check(rc, "conv_halo");
  return true;
}
// stride 2: `ntaps` (4) taps per parity class, `taps` (4 x 4) packed tap words (ops/functional.py conv_s2_dgrad_taps)
bool conv_igemm_dgrad_s2(const at::Tensor& dy, const at::Tensor& w, at::Tensor dx, int64_t kh, int64_t kw,
                         const std::vector<int64_t>& ntaps, const std::vector<int64_t>& taps, int64_t force_bn) {
  CHECK_CUDA(dy); CHECK_CUDA(w); CHECK_CUDA(dx);
  TORCH_CHECK(dy.scalar_type() == at::kBFloat16 && w.scalar_type() == at::kBFloat16 && dx.scalar_type() == at::kBFloat16 &&
              dy.dim() == 4 && dx.dim() == 4 && dy.is_contiguous() && w.is_contiguous() && dx.is_contiguous());
  TORCH_CHECK(ntaps.size() == 4 && taps.size() == 16, "conv_igemm_dgrad_s2: 4 classes x 4 taps");
  int nt[4], tw[16];
  for (int i = 0; i < 4; ++i) nt[i] = static_cast<int>(ntaps[i]);
  for (int i = 0; i < 16; ++i) tw[i] = static_cast<int>(taps[i]);
  const c10::cuda::CUDAGuard guard(dy.device());
  const int rc = b200_conv_igemm_dgrad_s2(cptr(dy), cptr(w), ptr(dx), static_cast<int>(dx.size(0)),
                                          static_cast<int>(dx.size(1)), static_cast<int>(dx.size(2)),
                                          static_cast<int>(dx.size(3)), static_cast<int>(dy.size(3)), static_cast<int>(kh),
                                          static_cast<int>(kw), static_cast<int>(dy.size(1)), static_cast<int>(dy.size(2)),
                                          nt, tw, static_cast<int>(force_bn), cur_stream());
  if (rc == -2) return false;
  check(rc, "conv_igemm_dgrad_s2");
  return true;
}
bool conv_igemm_wgrad(const at::Tensor& dy, const at::Tensor& x, at::Tensor dw, int64_t cout, int64_t kh, int64_t kw,
                      int64_t stride, int64_t pad, int64_t ho, int64_t wo, int64_t split_k, int64_t force_bn,
                      const std::optional<at::Tensor>& sgd_theta, const std::optional<at::Tensor>& sgd_theta_bf16,
                      const std::optional<at::Tensor>& sgd_mom, const std::optional<at::Tensor>& sgd_hyper,
                      bool sgd_nesterov, const std::optional<at::Tensor>& sgd_anchor,
                      const std::optional<at::Tensor>& sgd_corr, const std::optional<at::Tensor>& sgd_v) {
  CHECK_CUDA(dy); CHECK_CUDA(x); CHECK_CUDA(dw);
  TORCH_CHECK(x.scalar_type() == at::kBFloat16 && dy.scalar_type() == at::kBFloat16 && dw.scalar_type() == at::kFloat &&
              x.dim() == 4 && x.is_contiguous() && dy.is_contiguous());
  const c10::cuda::CUDAGuard guard(x.device());
  const std::optional<B200SgdEpilogue> sgd =
      sgd_epilogue(sgd_theta, sgd_theta_bf16, sgd_mom, sgd_hyper, sgd_nesterov, sgd_anchor, sgd_corr, sgd_v);
  const int rc = b200_conv_igemm_wgrad(cptr(dy), cptr(x), dw.data_ptr<float>(), static_cast<int>(x.size(0)),
                                       static_cast<int>(x.size(1)), static_cast<int>(x.size(2)), static_cast<int>(x.size(3)),
                                       static_cast<int>(cout), static_cast<int>(kh), static_cast<int>(kw),
                                       static_cast<int>(stride), static_cast<int>(pad), static_cast<int>(ho),
                                       static_cast<int>(wo), static_cast<int>(split_k), static_cast<int>(force_bn),
                                       sgd ? &*sgd : nullptr, cur_stream());
  if (rc == -2 || rc == B200_SGD_EPILOGUE_DECLINED) return false;
  check(rc, "conv_igemm_wgrad");
  return true;
}

void gemm_fp8(const at::Tensor& a, const at::Tensor& b, at::Tensor d, const std::optional<at::Tensor>& bias,
              const std::optional<at::Tensor>& sfa, const std::optional<at::Tensor>& sfb, int64_t M, int64_t N, int64_t K,
              int64_t lda, int64_t ldb, int64_t ldd, int64_t act, int64_t split_k, bool accumulate, double alpha) {
  CHECK_CUDA(a); CHECK_CUDA(b); CHECK_CUDA(d);
  TORCH_CHECK(a.element_size() == 1 && b.element_size() == 1, "gemm_fp8 operands must be 1-byte (e4m3)");
  const c10::cuda::CUDAGuard guard(a.device());
  check(b200_gemm_fp8(cptr(a), cptr(b), ptr(d), opt_ptr<const float>(bias), opt_ptr<const void>(sfa),
                      opt_ptr<const void>(sfb), M, N, K, lda, ldb, ldd, d.scalar_type() == at::kFloat, act, split_k,
                      accumulate, static_cast<float>(alpha), cur_stream()),
        "gemm_fp8");
}
void quant_mx_rows(const at::Tensor& x, at::Tensor q, at::Tensor sf, int64_t R, int64_t C, int64_t ld_in, int64_t Cp) {
  CHECK_CUDA(x);
  const c10::cuda::CUDAGuard guard(x.device());
  check(b200_quant_mx_rows(x.data_ptr(), q.data_ptr(), sf.data_ptr(), R, C, ld_in, Cp, cur_stream()), "quant_mx_rows");
}
void quant_mx_cols(const at::Tensor& x, at::Tensor q, at::Tensor sf, int64_t R, int64_t C, int64_t ld_in, int64_t Rp) {
  CHECK_CUDA(x);
  const c10::cuda::CUDAGuard guard(x.device());
  check(b200_quant_mx_cols(x.data_ptr(), q.data_ptr(), sf.data_ptr(), R, C, ld_in, Rp, cur_stream()), "quant_mx_cols");
}
void dequant_mx(const at::Tensor& q, const at::Tensor& sf, at::Tensor out, int64_t R, int64_t C, int64_t Cp) {
  CHECK_CUDA(q);
  const c10::cuda::CUDAGuard guard(q.device());
  check(b200_dequant_mx(q.data_ptr(), sf.data_ptr(), out.data_ptr<float>(), R, C, Cp, cur_stream()), "dequant_mx");
}

void fused_sgd(at::Tensor w, at::Tensor g, const std::optional<at::Tensor>& mom, const std::optional<at::Tensor>& wb,
               const at::Tensor& hyper, bool zero_grad, bool nesterov, const std::optional<at::Tensor>& wire_slot,
               const std::optional<at::Tensor>& pack_global, const std::optional<at::Tensor>& pack_scale, int64_t n_pack,
               bool wire_fp32, const std::optional<at::Tensor>& prox_anchor_, const std::optional<at::Tensor>& corr,
               const std::optional<at::Tensor>& adam_v) {
  CHECK_CUDA(w);
  TORCH_CHECK(w.scalar_type() == at::kFloat && g.scalar_type() == at::kFloat && hyper.scalar_type() == at::kFloat);
  TORCH_CHECK(w.is_contiguous() && g.is_contiguous() && w.numel() == g.numel());
  const c10::cuda::CUDAGuard guard(w.device());
  const float* anchor = prox_anchor(prox_anchor_, w.numel(), hyper);
  const float* c = scaf_corr(corr, w.numel(), anchor);
  check(b200_fused_sgd(w.data_ptr<float>(), g.data_ptr<float>(), opt_ptr<float>(mom), opt_ptr<void>(wb), w.numel(),
                       hyper.data_ptr<float>(), zero_grad, nesterov,
                       reinterpret_cast<const unsigned long long*>(opt_ptr<const int64_t>(wire_slot)),
                       opt_ptr<const float>(pack_global), opt_ptr<const float>(pack_scale), n_pack, wire_fp32, anchor,
                       c, adam_v_ptr(adam_v, w.numel(), opt_ptr<float>(mom), hyper, anchor, c), cur_stream()),
        "fused_sgd");
}

// segments: int64 [n][3] device table {offset, length, kind} over the arena (see fused_sgd_segments_kernel)
void fused_sgd_segments(at::Tensor w, at::Tensor g, const std::optional<at::Tensor>& mom,
                        const std::optional<at::Tensor>& wb, const at::Tensor& segments, const at::Tensor& hyper,
                        bool nesterov, const std::optional<at::Tensor>& prox_anchor_,
                        const std::optional<at::Tensor>& corr, const std::optional<at::Tensor>& adam_v) {
  CHECK_CUDA(w); CHECK_CUDA(segments);
  TORCH_CHECK(w.scalar_type() == at::kFloat && g.scalar_type() == at::kFloat && hyper.scalar_type() == at::kFloat);
  TORCH_CHECK(segments.scalar_type() == at::kLong && segments.dim() == 2 && segments.size(1) == 3 &&
              segments.is_contiguous(), "segments: contiguous int64 [n, 3]");
  const c10::cuda::CUDAGuard guard(w.device());
  const float* anchor = prox_anchor(prox_anchor_, w.numel(), hyper);
  const float* c = scaf_corr(corr, g.numel(), anchor);
  check(b200_fused_sgd_segments(w.data_ptr<float>(), g.data_ptr<float>(), opt_ptr<float>(mom), opt_ptr<void>(wb),
                                reinterpret_cast<const long long*>(segments.data_ptr<int64_t>()),
                                static_cast<int>(segments.size(0)), hyper.data_ptr<float>(), nesterov, anchor, c,
                                adam_v_ptr(adam_v, g.numel(), opt_ptr<float>(mom), hyper, anchor, c), cur_stream()),
        "fused_sgd_segments");
}

// SCAFFOLD control variates over the parameters: every buffer fp32, contiguous, at least n elements
inline void check_cv(const at::Tensor& t, int64_t n) {
  CHECK_CUDA(t);
  TORCH_CHECK(t.scalar_type() == at::kFloat && t.is_contiguous() && t.numel() >= n,
              "scaffold: contiguous fp32 buffers covering the parameters");
}
void scaffold_corr(at::Tensor corr, const at::Tensor& c, const at::Tensor& ci) {
  const int64_t n = corr.numel();
  check_cv(corr, n); check_cv(c, n); check_cv(ci, n);
  const c10::cuda::CUDAGuard guard(corr.device());
  check(b200_scaffold_corr(corr.data_ptr<float>(), c.data_ptr<float>(), ci.data_ptr<float>(), n, cur_stream()),
        "scaffold_corr");
}
void scaffold_dc(at::Tensor up, at::Tensor ci, const at::Tensor& c, const at::Tensor& global_w, const at::Tensor& theta,
                 double inv_k_eta, bool first) {
  const int64_t n = up.numel();
  check_cv(up, n); check_cv(ci, n); check_cv(c, n); check_cv(global_w, n); check_cv(theta, n);
  const c10::cuda::CUDAGuard guard(up.device());
  check(b200_scaffold_dc(up.data_ptr<float>(), ci.data_ptr<float>(), c.data_ptr<float>(), global_w.data_ptr<float>(),
                         theta.data_ptr<float>(), n, static_cast<float>(inv_k_eta), first ? 1 : 0, cur_stream()),
        "scaffold_dc");
}

void fold_client(at::Tensor acc, at::Tensor theta, const at::Tensor& global_w, const std::optional<at::Tensor>& wb,
                 const std::optional<at::Tensor>& mom, double nk, int64_t mode, bool reset) {
  CHECK_CUDA(acc);
  TORCH_CHECK(acc.scalar_type() == at::kFloat && theta.scalar_type() == at::kFloat && global_w.scalar_type() == at::kFloat);
  TORCH_CHECK(acc.numel() == theta.numel() && theta.numel() == global_w.numel());
  const c10::cuda::CUDAGuard guard(acc.device());
  check(b200_fold_client(acc.data_ptr<float>(), theta.data_ptr<float>(), global_w.data_ptr<float>(), opt_ptr<void>(wb),
                         opt_ptr<float>(mom), mom.has_value() && mom->defined() ? mom->numel() : 0, theta.numel(),
                         static_cast<float>(nk), static_cast<int>(mode), reset, cur_stream()),
        "fold_client");
}

void weighted_sum(at::Tensor dst, const std::vector<at::Tensor>& srcs, const std::vector<double>& weights) {
  CHECK_CUDA(dst);
  TORCH_CHECK(srcs.size() == weights.size() && !srcs.empty() && srcs.size() <= B200_MAX_RANKS);
  TORCH_CHECK(dst.is_contiguous());
  const c10::cuda::CUDAGuard guard(dst.device());
  std::vector<const void*> ps;
  std::vector<float> ws;
  for (size_t i = 0; i < srcs.size(); ++i) {
    TORCH_CHECK(srcs[i].is_cuda() && srcs[i].is_contiguous() && srcs[i].scalar_type() == dst.scalar_type() &&
                srcs[i].numel() == dst.numel());
    ps.push_back(srcs[i].data_ptr());
    ws.push_back(static_cast<float>(weights[i]));
  }
  const int dt = dst.scalar_type() == at::kBFloat16 ? 1 : 0;
  TORCH_CHECK(dt == 1 || dst.scalar_type() == at::kFloat, "weighted_sum supports fp32/bf16");
  check(b200_weighted_sum(dst.data_ptr(), ps.data(), ws.data(), static_cast<int>(ps.size()), dst.numel(), dt,
                          cur_stream()),
        "weighted_sum");
}

void cast(const at::Tensor& src, at::Tensor dst) {
  CHECK_CUDA(src);
  TORCH_CHECK(src.is_contiguous() && dst.is_contiguous() && src.numel() == dst.numel());
  const c10::cuda::CUDAGuard guard(src.device());
  if (src.scalar_type() == at::kFloat && dst.scalar_type() == at::kBFloat16)
    check(b200_cast_f32_bf16(src.data_ptr<float>(), dst.data_ptr(), src.numel(), cur_stream()), "cast");
  else if (src.scalar_type() == at::kBFloat16 && dst.scalar_type() == at::kFloat)
    check(b200_cast_bf16_f32(src.data_ptr(), dst.data_ptr<float>(), src.numel(), cur_stream()), "cast");
  else
    TORCH_CHECK(false, "cast: unsupported dtype pair");
}

void gather_rows(const at::Tensor& src, const at::Tensor& idx, at::Tensor dst) {
  CHECK_CUDA(src);
  TORCH_CHECK(idx.scalar_type() == at::kLong && src.is_contiguous() && dst.is_contiguous());
  const c10::cuda::CUDAGuard guard(src.device());
  const int64_t n = idx.numel();
  if (src.scalar_type() == at::kLong && src.dim() == 1) {
    check(b200_gather_rows_i64(src.data_ptr<int64_t>() ? reinterpret_cast<const long long*>(src.data_ptr<int64_t>()) : nullptr,
                               reinterpret_cast<const long long*>(idx.data_ptr<int64_t>()),
                               reinterpret_cast<long long*>(dst.data_ptr<int64_t>()), n, cur_stream()),
          "gather_i64");
    return;
  }
  const int64_t row_bytes = src.numel() / src.size(0) * src.element_size();
  check(b200_gather_rows(src.data_ptr(), reinterpret_cast<const long long*>(idx.data_ptr<int64_t>()), dst.data_ptr(), n,
                         row_bytes, cur_stream()),
        "gather_rows");
}

void colsum(const at::Tensor& x, at::Tensor out, int64_t rows, int64_t cols, bool accumulate) {
  CHECK_CUDA(x);
  const c10::cuda::CUDAGuard guard(x.device());
  check(b200_colsum(x.data_ptr(), out.data_ptr<float>(), rows, cols, accumulate, cur_stream()), "colsum");
}
void add_bf16(const at::Tensor& a, const at::Tensor& b, at::Tensor o, bool relu) {
  CHECK_CUDA(a);
  const c10::cuda::CUDAGuard guard(a.device());
  check(b200_add_bf16(a.data_ptr(), b.data_ptr(), o.data_ptr(), a.numel(), relu, cur_stream()), "add_bf16");
}
void relu_bwd(const at::Tensor& y, const at::Tensor& dy, at::Tensor dx) {
  CHECK_CUDA(y);
  const c10::cuda::CUDAGuard guard(y.device());
  check(b200_relu_bwd_bf16(y.data_ptr(), dy.data_ptr(), dx.data_ptr(), y.numel(), cur_stream()), "relu_bwd");
}
void gelu(const at::Tensor& x, at::Tensor y) {
  CHECK_CUDA(x);
  const c10::cuda::CUDAGuard guard(x.device());
  check(b200_gelu_bf16(x.data_ptr(), y.data_ptr(), x.numel(), cur_stream()), "gelu");
}
void gelu_bwd(const at::Tensor& x, const at::Tensor& dy, at::Tensor dx) {
  CHECK_CUDA(x);
  const c10::cuda::CUDAGuard guard(x.device());
  check(b200_gelu_bwd_bf16(x.data_ptr(), dy.data_ptr(), dx.data_ptr(), x.numel(), cur_stream()), "gelu_bwd");
}
void embedding_bwd(const at::Tensor& dy, const at::Tensor& idx, at::Tensor grad) {
  CHECK_CUDA(dy);
  TORCH_CHECK(dy.scalar_type() == at::kBFloat16 && grad.scalar_type() == at::kFloat && idx.scalar_type() == at::kLong);
  const c10::cuda::CUDAGuard guard(dy.device());
  check(b200_embedding_bwd(dy.data_ptr(), reinterpret_cast<const long long*>(idx.data_ptr<int64_t>()),
                           grad.data_ptr<float>(), idx.numel(), static_cast<int>(dy.size(-1)), cur_stream()),
        "embedding_bwd");
}
void pad_rows(const at::Tensor& s, at::Tensor d, int64_t rows, int64_t k, int64_t kp,
              const std::optional<at::Tensor>& flags, const std::optional<at::Tensor>& epoch_word, int64_t elem_off,
              int64_t granule) {
  CHECK_CUDA(s);
  const c10::cuda::CUDAGuard guard(s.device());
  check(b200_pad_rows_bf16(s.data_ptr(), d.data_ptr(), rows, k, kp, opt_ptr<const uint32_t>(flags),
                           opt_ptr<const uint32_t>(epoch_word), elem_off, static_cast<int>(granule), cur_stream()),
        "pad_rows");
}

// ---- fused FedAvg collective -------------------------------------------------------------------
// the arguments every variant of the collective shares
static void fill_fedavg_args(FedAvgArgs& a, const std::vector<int64_t>& wire_ptrs, const std::vector<int64_t>& pad_ptrs,
                             int64_t wire_mc, at::Tensor& theta, const std::optional<at::Tensor>& global_w,
                             const std::optional<at::Tensor>& theta_bf16, const std::optional<at::Tensor>& momentum,
                             const std::optional<at::Tensor>& int_local, const std::vector<int64_t>& int_wire_ptrs,
                             const std::optional<at::Tensor>& loss_local, const std::vector<int64_t>& loss_wire_ptrs,
                             const std::optional<at::Tensor>& loss_out, const std::vector<double>& n_samples,
                             bool counts_from_flags, int64_t alive_mask, int64_t rank, int64_t world, int64_t wire_kind,
                             bool delta, bool use_nvls, int64_t epoch, const std::optional<at::Tensor>& tile_flags,
                             int64_t flag_value, int64_t tile_elems, int64_t timeout_log2,
                             const std::optional<at::Tensor>& status, const std::optional<at::Tensor>& phase_ns,
                             bool prepacked) {
  CHECK_CUDA(theta);
  TORCH_CHECK(world <= B200_MAX_RANKS && static_cast<int64_t>(wire_ptrs.size()) == world &&
              static_cast<int64_t>(pad_ptrs.size()) == world && static_cast<int64_t>(n_samples.size()) == world);
  TORCH_CHECK(theta.scalar_type() == at::kFloat && theta.is_contiguous());
  for (int64_t k = 0; k < world; ++k) {
    a.wire[k] = reinterpret_cast<void*>(wire_ptrs[k]);
    a.pads[k] = reinterpret_cast<unsigned long long*>(pad_ptrs[k]);
    a.n_samples[k] = static_cast<float>(n_samples[k]);
    a.int_wire[k] = k < static_cast<int64_t>(int_wire_ptrs.size()) ? reinterpret_cast<long long*>(int_wire_ptrs[k]) : nullptr;
    a.loss_wire[k] = k < static_cast<int64_t>(loss_wire_ptrs.size()) ? reinterpret_cast<float*>(loss_wire_ptrs[k]) : nullptr;
  }
  a.wire_mc = reinterpret_cast<void*>(wire_mc);
  a.theta = theta.data_ptr<float>();
  a.global_w = opt_ptr<float>(global_w);
  a.theta_bf16 = opt_ptr<void>(theta_bf16);
  a.momentum = opt_ptr<float>(momentum);
  a.n_momentum = a.momentum != nullptr ? momentum->numel() : 0;
  a.int_local = opt_ptr<long long>(int_local);
  a.n_int = (a.int_local != nullptr && !int_wire_ptrs.empty()) ? static_cast<int>(int_local->numel()) : 0;
  a.loss_local = opt_ptr<float>(loss_local);
  a.loss_out = opt_ptr<float>(loss_out);
  a.n_loss = (a.loss_local != nullptr && !loss_wire_ptrs.empty()) ? static_cast<int>(loss_local->numel()) : 0;
  a.counts_from_flags = counts_from_flags;
  a.nvls_prescale = 1.0f;
  a.alive_mask = static_cast<uint32_t>(alive_mask);
  a.rank = static_cast<int>(rank);
  a.world = static_cast<int>(world);
  a.n = theta.numel();
  a.wire_kind = static_cast<int>(wire_kind);
  a.delta = delta;
  a.use_nvls = use_nvls;
  a.epoch = static_cast<uint32_t>(epoch);
  a.tile_flags = opt_ptr<uint32_t>(tile_flags);
  a.flag_value = static_cast<uint32_t>(flag_value);
  a.tile_elems = static_cast<int>(tile_elems);
  a.timeout_log2 = static_cast<int>(timeout_log2);
  a.prepacked = prepacked ? 1 : 0;
  a.status = opt_ptr<int>(status);
  a.phase_ns = nullptr;
  if (phase_ns.has_value()) {
    TORCH_CHECK(phase_ns->scalar_type() == at::kLong && phase_ns->numel() >= 16, "phase_ns: int64[16]");
    a.phase_ns = reinterpret_cast<unsigned long long*>(phase_ns->data_ptr<int64_t>());
  }
}

void fedavg_allreduce(const std::vector<int64_t>& wire_ptrs, const std::vector<int64_t>& pad_ptrs, int64_t wire_mc,
                      at::Tensor theta, const std::optional<at::Tensor>& global_w,
                      const std::optional<at::Tensor>& theta_bf16, const std::optional<at::Tensor>& momentum,
                      const std::optional<at::Tensor>& int_local, const std::vector<int64_t>& int_wire_ptrs,
                      const std::optional<at::Tensor>& loss_local, const std::vector<int64_t>& loss_wire_ptrs,
                      const std::optional<at::Tensor>& loss_out, const std::vector<double>& n_samples,
                      bool counts_from_flags, int64_t alive_mask, int64_t rank, int64_t world, int64_t wire_kind,
                      bool delta, bool use_nvls, int64_t epoch, const std::optional<at::Tensor>& tile_flags,
                      int64_t flag_value, int64_t tile_elems, int64_t n_ctas, int64_t timeout_log2,
                      const std::optional<at::Tensor>& status, const std::optional<at::Tensor>& phase_ns, bool prepacked,
                      const std::vector<int64_t>& clip_page_ptrs, double dp_noise_std, int64_t dp_seed, int64_t dp_round,
                      const std::optional<at::Tensor>& scaf_dc, const std::optional<at::Tensor>& scaf_c,
                      int64_t scaf_seg1_off, double scaf_inv_clients) {
  FedAvgDPArgs a = {};
  fill_fedavg_args(a, wire_ptrs, pad_ptrs, wire_mc, theta, global_w, theta_bf16, momentum, int_local, int_wire_ptrs,
                   loss_local, loss_wire_ptrs, loss_out, n_samples, counts_from_flags, alive_mask, rank, world, wire_kind,
                   delta, use_nvls, epoch, tile_flags, flag_value, tile_elems, timeout_log2, status, phase_ns, prepacked);
  const c10::cuda::CUDAGuard guard(theta.device());
  // DP-FedAvg: one clip page per rank (empty = off); the seed is the 64-bit Philox key, passed as its int64 bit pattern
  const bool dp = !clip_page_ptrs.empty();
  if (dp) {
    TORCH_CHECK(static_cast<int64_t>(clip_page_ptrs.size()) == world, "DP: one clip page per rank");
    for (int64_t k = 0; k < world; ++k) a.clip_page[k] = reinterpret_cast<const float*>(clip_page_ptrs[k]);
    a.noise_std = static_cast<float>(dp_noise_std);
    a.seed = static_cast<unsigned long long>(dp_seed);
    a.round = static_cast<uint32_t>(dp_round);
    TORCH_CHECK(delta && !use_nvls, "DP needs delta mode on peer loads");
  }
  TORCH_CHECK(!delta || a.global_w != nullptr, "delta mode needs the global copy");
  TORCH_CHECK(!use_nvls || a.wire_mc != nullptr, "NVLS mode needs the multicast address");
  // SCAFFOLD: the control-variate segment (dc in, c updated) rides in the same launch
  if (scaf_c.has_value() && scaf_c->defined()) {
    TORCH_CHECK(!dp && delta && !use_nvls, "SCAFFOLD rounds need delta mode on peer loads, without DP");
    TORCH_CHECK(scaf_dc.has_value() && scaf_dc->defined(), "SCAFFOLD: dc and c go together");
    check_cv(*scaf_c, scaf_c->numel());
    check_cv(*scaf_dc, scaf_c->numel());
    FedAvgScaffoldArgs sa = {};
    static_cast<FedAvgArgs&>(sa) = static_cast<const FedAvgArgs&>(a);
    sa.dc = scaf_dc->data_ptr<float>();
    sa.c = scaf_c->data_ptr<float>();
    sa.n_c = scaf_c->numel();
    sa.seg1_off = scaf_seg1_off;
    sa.inv_clients = static_cast<float>(scaf_inv_clients);
    check(b200_fedavg_allreduce_scaffold(&sa, static_cast<int>(n_ctas), cur_stream()), "fedavg_allreduce");
    return;
  }
  check(dp ? b200_fedavg_allreduce_dp(&a, static_cast<int>(n_ctas), cur_stream())
           : b200_fedavg_allreduce(&a, static_cast<int>(n_ctas), cur_stream()),
        "fedavg_allreduce");
}

// robust round: seg_page_ptrs = every rank's count page, trim_b = floor(beta * P) for P = 0 .. 32 (trimmed mean)
void fedavg_allreduce_robust(const std::vector<int64_t>& wire_ptrs, const std::vector<int64_t>& pad_ptrs,
                             at::Tensor theta, const at::Tensor& global_w, const std::optional<at::Tensor>& theta_bf16,
                             const std::optional<at::Tensor>& momentum, const std::optional<at::Tensor>& int_local,
                             const std::vector<int64_t>& int_wire_ptrs, const std::optional<at::Tensor>& loss_local,
                             const std::vector<int64_t>& loss_wire_ptrs, const std::optional<at::Tensor>& loss_out,
                             const std::vector<double>& n_samples, bool counts_from_flags, int64_t alive_mask, int64_t rank,
                             int64_t world, int64_t wire_kind, int64_t epoch, int64_t tile_elems, int64_t n_ctas,
                             int64_t timeout_log2, const std::optional<at::Tensor>& status,
                             const std::optional<at::Tensor>& phase_ns, bool prepacked,
                             const std::vector<int64_t>& seg_page_ptrs, int64_t my_segs, int64_t seg_stride, int64_t kind,
                             const std::vector<int64_t>& trim_b) {
  FedAvgRobustArgs a = {};
  fill_fedavg_args(a, wire_ptrs, pad_ptrs, 0, theta, global_w, theta_bf16, momentum, int_local, int_wire_ptrs, loss_local,
                   loss_wire_ptrs, loss_out, n_samples, counts_from_flags, alive_mask, rank, world, wire_kind, true, false,
                   epoch, std::nullopt, 0, tile_elems, timeout_log2, status, phase_ns, prepacked);
  TORCH_CHECK(static_cast<int64_t>(seg_page_ptrs.size()) == world, "robust: one count page per rank");
  TORCH_CHECK(static_cast<int64_t>(trim_b.size()) == B200_MAX_ROBUST_CLIENTS + 1, "robust: trim_b for P = 0 .. 32");
  TORCH_CHECK(my_segs >= 0 && my_segs <= B200_MAX_ROBUST_CLIENTS, "robust: at most 32 segments per rank");
  for (int64_t k = 0; k < world; ++k) a.seg_page[k] = reinterpret_cast<uint32_t*>(seg_page_ptrs[k]);
  for (int p = 0; p <= B200_MAX_ROBUST_CLIENTS; ++p) {
    TORCH_CHECK(trim_b[p] >= 0 && 2 * trim_b[p] < (p > 0 ? p : 1), "robust: need P - 2b >= 1");
    a.trim_b[p] = static_cast<uint8_t>(trim_b[p]);
  }
  a.my_segs = static_cast<uint32_t>(my_segs);
  a.seg_stride = seg_stride;
  a.kind = static_cast<int>(kind);
  const c10::cuda::CUDAGuard guard(theta.device());
  check(b200_fedavg_allreduce_robust(&a, static_cast<int>(n_ctas), cur_stream()), "fedavg_allreduce_robust");
}

// one logical client's wire segment at address seg (see b200_pack_client)
void pack_client(int64_t seg, at::Tensor theta, const at::Tensor& global_w, const std::optional<at::Tensor>& wb,
                 const std::optional<at::Tensor>& mom, int64_t wire_kind, bool reset) {
  CHECK_CUDA(theta);
  TORCH_CHECK(theta.scalar_type() == at::kFloat && global_w.scalar_type() == at::kFloat && theta.is_contiguous() &&
              global_w.is_contiguous() && global_w.numel() == theta.numel(), "pack_client: fp32 theta / global_w");
  const c10::cuda::CUDAGuard guard(theta.device());
  check(b200_pack_client(reinterpret_cast<void*>(seg), theta.data_ptr<float>(), global_w.data_ptr<float>(),
                         opt_ptr<void>(wb), opt_ptr<float>(mom), mom.has_value() && mom->defined() ? mom->numel() : 0,
                         theta.numel(), static_cast<int>(wire_kind), reset ? 1 : 0, cur_stream()),
        "pack_client");
}

// DP clip factor of theta against global_w over theta's n elements; work: int64 [DP_WORK_WORDS], zeroed once
void dp_clip_factor(const at::Tensor& theta, const at::Tensor& global_w, double clip, at::Tensor work, at::Tensor s_out,
                    at::Tensor norm_out, int64_t s_copy, const std::optional<at::Tensor>& nonfinite) {
  CHECK_CUDA(theta); CHECK_CUDA(global_w); CHECK_CUDA(work); CHECK_CUDA(s_out); CHECK_CUDA(norm_out);
  TORCH_CHECK(theta.scalar_type() == at::kFloat && global_w.scalar_type() == at::kFloat && theta.is_contiguous() &&
              global_w.is_contiguous() && global_w.numel() >= theta.numel(), "dp_clip_factor: fp32 theta / global_w");
  TORCH_CHECK(work.scalar_type() == at::kLong && work.numel() >= B200_DP_WORK_WORDS, "dp_clip_factor: int64 work");
  TORCH_CHECK(s_out.scalar_type() == at::kFloat && norm_out.scalar_type() == at::kFloat && s_out.numel() >= 1 &&
              norm_out.numel() >= 1, "dp_clip_factor: fp32 outputs");
  TORCH_CHECK(!nonfinite.has_value() || nonfinite->scalar_type() == at::kInt, "dp_clip_factor: int32 counter");
  const c10::cuda::CUDAGuard guard(theta.device());
  check(b200_dp_clip_factor(theta.data_ptr<float>(), global_w.data_ptr<float>(), theta.numel(), static_cast<float>(clip),
                            work.data_ptr(), s_out.data_ptr<float>(), norm_out.data_ptr<float>(),
                            reinterpret_cast<float*>(s_copy), opt_ptr<int>(nonfinite), cur_stream()),
        "dp_clip_factor");
}

void fold_client_scaled(at::Tensor acc, at::Tensor theta, const at::Tensor& global_w, const std::optional<at::Tensor>& wb,
                        const std::optional<at::Tensor>& mom, const at::Tensor& s, bool first, bool reset) {
  CHECK_CUDA(acc); CHECK_CUDA(s);
  TORCH_CHECK(acc.scalar_type() == at::kFloat && theta.scalar_type() == at::kFloat && global_w.scalar_type() == at::kFloat &&
              s.scalar_type() == at::kFloat && s.numel() >= 1);
  TORCH_CHECK(acc.numel() == theta.numel() && theta.numel() == global_w.numel());
  const c10::cuda::CUDAGuard guard(acc.device());
  check(b200_fold_client_scaled(acc.data_ptr<float>(), theta.data_ptr<float>(), global_w.data_ptr<float>(),
                                opt_ptr<void>(wb), opt_ptr<float>(mom), mom.has_value() && mom->defined() ? mom->numel() : 0,
                                theta.numel(), s.data_ptr<float>(), first, reset, cur_stream()),
        "fold_client_scaled");
}

void flag_barrier(const std::vector<int64_t>& pad_ptrs, int64_t rank, int64_t world, int64_t alive_mask, int64_t epoch,
                  int64_t slot) {
  std::vector<unsigned long long*> pads;
  for (auto p : pad_ptrs) pads.push_back(reinterpret_cast<unsigned long long*>(p));
  check(b200_flag_barrier(pads.data(), rank, world, static_cast<uint32_t>(alive_mask), static_cast<uint32_t>(epoch), slot,
                          cur_stream()),
        "flag_barrier");
}

// ---- conv plumbing -------------------------------------------------------------------------------
void im2col(const at::Tensor& x, at::Tensor col, int64_t N, int64_t H, int64_t W, int64_t C, int64_t KH, int64_t KW,
            int64_t stride, int64_t pad, int64_t Ho, int64_t Wo, int64_t kp) {
  CHECK_CUDA(x);
  const c10::cuda::CUDAGuard guard(x.device());
  check(b200_im2col_nhwc(x.data_ptr(), col.data_ptr(), N, H, W, C, KH, KW, stride, pad, Ho, Wo, kp, cur_stream()),
        "im2col");
}
void col2im(const at::Tensor& col, at::Tensor dx, int64_t N, int64_t H, int64_t W, int64_t C, int64_t KH, int64_t KW,
            int64_t stride, int64_t pad, int64_t Ho, int64_t Wo, int64_t kp) {
  CHECK_CUDA(col);
  const c10::cuda::CUDAGuard guard(col.device());
  check(b200_col2im_nhwc(col.data_ptr(), dx.data_ptr(), N, H, W, C, KH, KW, stride, pad, Ho, Wo, kp, cur_stream()),
        "col2im");
}
void maxpool(const at::Tensor& x, at::Tensor y, at::Tensor arg, int64_t N, int64_t H, int64_t W, int64_t C, int64_t k,
             int64_t stride, int64_t pad, int64_t Ho, int64_t Wo) {
  CHECK_CUDA(x);
  const c10::cuda::CUDAGuard guard(x.device());
  const int u8 = arg.scalar_type() == at::kByte;      // byte-sized winners: the 16-byte kernels
  check(b200_maxpool_nhwc(x.data_ptr(), y.data_ptr(), reinterpret_cast<int*>(arg.data_ptr()), N, H, W, C, k, stride, pad,
                          Ho, Wo, u8, cur_stream()),
        "maxpool");
}
void maxpool_bwd(const at::Tensor& dy, const std::optional<at::Tensor>& dy_b, const at::Tensor& arg, at::Tensor dx,
                 int64_t N, int64_t H, int64_t W, int64_t C, int64_t Ho, int64_t Wo, int64_t k, int64_t stride, int64_t pad) {
  CHECK_CUDA(dy);
  const c10::cuda::CUDAGuard guard(dy.device());
  const int u8 = arg.scalar_type() == at::kByte;
  check(b200_maxpool_bwd_nhwc(dy.data_ptr(), opt_ptr<const void>(dy_b), reinterpret_cast<const int*>(arg.data_ptr()),
                              dx.data_ptr(), N, H, W, C, Ho, Wo, k, stride, pad, u8, cur_stream()),
        "maxpool_bwd");
}
void avgpool(const at::Tensor& x, at::Tensor y, int64_t N, int64_t HW, int64_t C) {
  CHECK_CUDA(x);
  const c10::cuda::CUDAGuard guard(x.device());
  check(b200_avgpool_nhwc(x.data_ptr(), y.data_ptr(), N, HW, C, cur_stream()), "avgpool");
}
void avgpool_bwd(const at::Tensor& dy, at::Tensor dx, int64_t N, int64_t HW, int64_t C) {
  CHECK_CUDA(dy);
  const c10::cuda::CUDAGuard guard(dy.device());
  check(b200_avgpool_bwd_nhwc(dy.data_ptr(), dx.data_ptr(), N, HW, C, cur_stream()), "avgpool_bwd");
}

// ---- normalisation ---------------------------------------------------------------------------------
void bn_stats(const at::Tensor& x, at::Tensor sums, int64_t rows, int64_t C) {
  CHECK_CUDA(x);
  const c10::cuda::CUDAGuard guard(x.device());
  check(b200_bn_stats(x.data_ptr(), sums.data_ptr<float>(), rows, C, cur_stream()), "bn_stats");
}
void bn_apply(const at::Tensor& x, const std::optional<at::Tensor>& res, at::Tensor y, at::Tensor sums,
              const std::optional<at::Tensor>& gamma, const std::optional<at::Tensor>& beta,
              const std::optional<at::Tensor>& rmean, const std::optional<at::Tensor>& rvar, at::Tensor save_mean,
              at::Tensor save_rstd, const std::optional<at::Tensor>& nbt, int64_t rows, int64_t C, double eps,
              double momentum, bool relu, bool training) {
  CHECK_CUDA(x);
  const c10::cuda::CUDAGuard guard(x.device());
  check(b200_bn_apply(x.data_ptr(), opt_ptr<const void>(res), y.data_ptr(), sums.data_ptr<float>(),
                      opt_ptr<const float>(gamma), opt_ptr<const float>(beta), opt_ptr<float>(rmean),
                      opt_ptr<float>(rvar), save_mean.data_ptr<float>(), save_rstd.data_ptr<float>(),
                      opt_ptr<long long>(nbt), rows, C,
                      static_cast<float>(eps), static_cast<float>(momentum), relu, training, cur_stream()),
        "bn_apply");
}
void bn_bwd_reduce(const at::Tensor& x, const at::Tensor& y, const at::Tensor& dy, const at::Tensor& mean,
                   const at::Tensor& rstd, at::Tensor sums, int64_t rows, int64_t C, bool relu) {
  CHECK_CUDA(x);
  const c10::cuda::CUDAGuard guard(x.device());
  check(b200_bn_bwd_reduce(x.data_ptr(), y.data_ptr(), dy.data_ptr(), mean.data_ptr<float>(), rstd.data_ptr<float>(),
                           sums.data_ptr<float>(), rows, C, relu, cur_stream()),
        "bn_bwd_reduce");
}
void bn_bwd_apply(const at::Tensor& x, const at::Tensor& y, const at::Tensor& dy, at::Tensor dx,
                  const std::optional<at::Tensor>& dres, const std::optional<at::Tensor>& gamma, const at::Tensor& mean,
                  const at::Tensor& rstd, at::Tensor sums, const std::optional<at::Tensor>& dgamma,
                  const std::optional<at::Tensor>& dbeta, int64_t rows, int64_t C, bool relu) {
  CHECK_CUDA(x);
  const c10::cuda::CUDAGuard guard(x.device());
  check(b200_bn_bwd_apply(x.data_ptr(), y.data_ptr(), dy.data_ptr(), dx.data_ptr(), opt_ptr<void>(dres),
                          opt_ptr<const float>(gamma), mean.data_ptr<float>(), rstd.data_ptr<float>(),
                          sums.data_ptr<float>(), opt_ptr<float>(dgamma), opt_ptr<float>(dbeta), rows, C, relu,
                          cur_stream()),
        "bn_bwd_apply");
}
// ResNet stem: BatchNorm + ReLU + max-pool in one pass (the normalised activation is never materialised) and its backward;
// false = shape not supported, use the separate kernels
bool bn_relu_maxpool(const at::Tensor& z, at::Tensor p, at::Tensor arg, at::Tensor sums,
                     const std::optional<at::Tensor>& gamma, const std::optional<at::Tensor>& beta,
                     const std::optional<at::Tensor>& rmean, const std::optional<at::Tensor>& rvar, at::Tensor save_mean,
                     at::Tensor save_rstd, const std::optional<at::Tensor>& nbt, int64_t N, int64_t H, int64_t W, int64_t C,
                     int64_t k, int64_t stride, int64_t pad, int64_t Ho, int64_t Wo, double eps, double momentum) {
  CHECK_CUDA(z);
  const c10::cuda::CUDAGuard guard(z.device());
  const int rc = b200_bn_relu_maxpool(z.data_ptr(), p.data_ptr(), arg.data_ptr(), sums.data_ptr<float>(),
                                      opt_ptr<const float>(gamma), opt_ptr<const float>(beta), opt_ptr<float>(rmean),
                                      opt_ptr<float>(rvar), save_mean.data_ptr<float>(), save_rstd.data_ptr<float>(),
                                      opt_ptr<long long>(nbt), static_cast<int>(N), static_cast<int>(H), static_cast<int>(W),
                                      static_cast<int>(C), static_cast<int>(k), static_cast<int>(stride),
                                      static_cast<int>(pad), static_cast<int>(Ho), static_cast<int>(Wo),
                                      static_cast<float>(eps), static_cast<float>(momentum), cur_stream());
  if (rc == -2) return false;
  check(rc, "bn_relu_maxpool");
  return true;
}
bool bn_maxpool_bwd(const at::Tensor& z, const at::Tensor& p, const at::Tensor& arg, const at::Tensor& dy_a,
                    const std::optional<at::Tensor>& dy_b, at::Tensor dz, const std::optional<at::Tensor>& gamma,
                    const at::Tensor& mean, const at::Tensor& rstd, at::Tensor sums, const std::optional<at::Tensor>& dgamma,
                    const std::optional<at::Tensor>& dbeta, int64_t N, int64_t H, int64_t W, int64_t C, int64_t k,
                    int64_t stride, int64_t pad, int64_t Ho, int64_t Wo) {
  CHECK_CUDA(z);
  const c10::cuda::CUDAGuard guard(z.device());
  const int rc = b200_bn_maxpool_bwd(z.data_ptr(), p.data_ptr(), arg.data_ptr(), dy_a.data_ptr(), opt_ptr<const void>(dy_b),
                                     dz.data_ptr(), opt_ptr<const float>(gamma), mean.data_ptr<float>(),
                                     rstd.data_ptr<float>(), sums.data_ptr<float>(), opt_ptr<float>(dgamma),
                                     opt_ptr<float>(dbeta), static_cast<int>(N), static_cast<int>(H), static_cast<int>(W),
                                     static_cast<int>(C), static_cast<int>(k), static_cast<int>(stride),
                                     static_cast<int>(pad), static_cast<int>(Ho), static_cast<int>(Wo), cur_stream());
  if (rc == -2) return false;
  check(rc, "bn_maxpool_bwd");
  return true;
}
// single-kernel BatchNorm backward (cluster per channel slice); dy = dy_a (+ dy_b).  False: shape not supported.
bool bn_bwd_cluster(const at::Tensor& x, const at::Tensor& y, const at::Tensor& dy_a, const std::optional<at::Tensor>& dy_b,
                    at::Tensor dx, const std::optional<at::Tensor>& dres, const std::optional<at::Tensor>& gamma,
                    const at::Tensor& mean, const at::Tensor& rstd, const std::optional<at::Tensor>& dgamma,
                    const std::optional<at::Tensor>& dbeta, int64_t rows, int64_t C, bool relu, int64_t max_cluster) {
  CHECK_CUDA(x);
  const c10::cuda::CUDAGuard guard(x.device());
  const int rc = b200_bn_bwd_cluster(x.data_ptr(), y.data_ptr(), dy_a.data_ptr(), opt_ptr<const void>(dy_b), dx.data_ptr(),
                                     opt_ptr<void>(dres), opt_ptr<const float>(gamma), mean.data_ptr<float>(),
                                     rstd.data_ptr<float>(), opt_ptr<float>(dgamma), opt_ptr<float>(dbeta), rows, C, relu,
                                     static_cast<int>(max_cluster), cur_stream());
  if (rc == -2) return false;
  check(rc, "bn_bwd_cluster");
  return true;
}
// eval-mode BatchNorm folding of every BatchNorm in `table` (int64 [n_bn, 7], see launch.h) into `out`
void bn_fold_eval(const at::Tensor& arena, const at::Tensor& table, at::Tensor out) {
  CHECK_CUDA(arena); CHECK_CUDA(table); CHECK_CUDA(out);
  TORCH_CHECK(arena.scalar_type() == at::kFloat && out.scalar_type() == at::kFloat && table.scalar_type() == at::kLong &&
                  table.dim() == 2 && table.size(1) == 7 && table.is_contiguous() && out.is_contiguous(),
              "bn_fold_eval: fp32 arena / out, int64 [n, 7] table");
  const c10::cuda::CUDAGuard guard(arena.device());
  check(b200_bn_fold_eval(arena.data_ptr<float>(), reinterpret_cast<const long long*>(table.data_ptr<int64_t>()),
                          static_cast<int>(table.size(0)), out.data_ptr<float>(), cur_stream()),
        "bn_fold_eval");
}
void layernorm_fwd(const at::Tensor& x, const std::optional<at::Tensor>& res, at::Tensor y, const at::Tensor& gamma,
                   const at::Tensor& beta, at::Tensor mean, at::Tensor rstd, int64_t rows, int64_t C, double eps) {
  CHECK_CUDA(x);
  const c10::cuda::CUDAGuard guard(x.device());
  check(b200_layernorm_fwd(x.data_ptr(), opt_ptr<const void>(res), y.data_ptr(), gamma.data_ptr<float>(),
                           beta.data_ptr<float>(), mean.data_ptr<float>(), rstd.data_ptr<float>(), rows, C,
                           static_cast<float>(eps), cur_stream()),
        "layernorm_fwd");
}
void layernorm_bwd(const at::Tensor& x, const at::Tensor& dy, at::Tensor dx, const at::Tensor& gamma,
                   const at::Tensor& mean, const at::Tensor& rstd, at::Tensor dgamma, at::Tensor dbeta, int64_t rows,
                   int64_t C) {
  CHECK_CUDA(x);
  const c10::cuda::CUDAGuard guard(x.device());
  check(b200_layernorm_bwd(x.data_ptr(), dy.data_ptr(), dx.data_ptr(), gamma.data_ptr<float>(), mean.data_ptr<float>(),
                           rstd.data_ptr<float>(), dgamma.data_ptr<float>(), dbeta.data_ptr<float>(), rows, C,
                           cur_stream()),
        "layernorm_bwd");
}
void softmax_fwd(const at::Tensor& x, at::Tensor y, int64_t rows, int64_t C, double scale) {
  CHECK_CUDA(x);
  const c10::cuda::CUDAGuard guard(x.device());
  check(b200_softmax_fwd(x.data_ptr(), y.data_ptr(), rows, C, static_cast<float>(scale), cur_stream()), "softmax_fwd");
}
void softmax_bwd(const at::Tensor& y, const at::Tensor& dy, at::Tensor dx, int64_t rows, int64_t C, double scale) {
  CHECK_CUDA(y);
  const c10::cuda::CUDAGuard guard(y.device());
  check(b200_softmax_bwd(y.data_ptr(), dy.data_ptr(), dx.data_ptr(), rows, C, static_cast<float>(scale), cur_stream()),
        "softmax_bwd");
}

// ---- losses ------------------------------------------------------------------------------------------
void softmax_xent(const at::Tensor& logits, const at::Tensor& target, const std::optional<at::Tensor>& dlogits,
                  at::Tensor loss_acc, int64_t rows, int64_t C, int64_t ld, double grad_scale) {
  CHECK_CUDA(logits);
  TORCH_CHECK(target.scalar_type() == at::kLong && loss_acc.scalar_type() == at::kFloat && loss_acc.numel() >= 2);
  const c10::cuda::CUDAGuard guard(logits.device());
  const int in32 = logits.scalar_type() == at::kFloat;
  const int out32 = dlogits.has_value() && dlogits->defined() && dlogits->scalar_type() == at::kFloat;
  check(b200_softmax_xent(logits.data_ptr(), in32, reinterpret_cast<const long long*>(target.data_ptr<int64_t>()),
                          opt_ptr<void>(dlogits), out32, loss_acc.data_ptr<float>(), rows, C, ld,
                          static_cast<float>(grad_scale), cur_stream()),
        "softmax_xent");
}
// False: shape not supported by the one-launch head (more than 32 classes, K % 8, ...)
bool linear_xent_head(const at::Tensor& x, const at::Tensor& w, const std::optional<at::Tensor>& bias, const at::Tensor& target,
                      const std::optional<at::Tensor>& dx, at::Tensor dw, const std::optional<at::Tensor>& db,
                      at::Tensor loss_acc, const std::optional<at::Tensor>& logits_out, double grad_scale) {
  CHECK_CUDA(x);
  TORCH_CHECK(x.scalar_type() == at::kBFloat16 && w.scalar_type() == at::kBFloat16 && x.dim() == 2 && w.dim() == 2 &&
              x.is_contiguous() && w.is_contiguous() && x.size(1) == w.size(1));
  TORCH_CHECK(target.scalar_type() == at::kLong && dw.scalar_type() == at::kFloat && dw.is_contiguous() &&
              dw.numel() == w.numel() && loss_acc.scalar_type() == at::kFloat && loss_acc.numel() >= 2);
  const c10::cuda::CUDAGuard guard(x.device());
  const int rc = b200_linear_xent_head(x.data_ptr(), w.data_ptr(), opt_ptr<const float>(bias),
                                       reinterpret_cast<const long long*>(target.data_ptr<int64_t>()), opt_ptr<void>(dx),
                                       dw.data_ptr<float>(), opt_ptr<float>(db), loss_acc.data_ptr<float>(),
                                       opt_ptr<float>(logits_out), static_cast<int>(x.size(0)), static_cast<int>(x.size(1)),
                                       static_cast<int>(w.size(0)), static_cast<float>(grad_scale), cur_stream());
  if (rc == -2) return false;
  check(rc, "linear_xent_head");
  return true;
}
// forward-only classifier head (evaluation); false: shape not supported
bool linear_xent_eval(const at::Tensor& x, const at::Tensor& w, const std::optional<at::Tensor>& bias, const at::Tensor& target,
                      at::Tensor loss_acc, const std::optional<at::Tensor>& logits_out) {
  CHECK_CUDA(x);
  TORCH_CHECK(x.scalar_type() == at::kBFloat16 && w.scalar_type() == at::kBFloat16 && x.dim() == 2 && w.dim() == 2 &&
              x.is_contiguous() && w.is_contiguous() && x.size(1) == w.size(1));
  TORCH_CHECK(target.scalar_type() == at::kLong && target.numel() >= x.size(0) && loss_acc.scalar_type() == at::kFloat &&
              loss_acc.numel() >= 2);
  TORCH_CHECK(!bias.has_value() || (bias->scalar_type() == at::kFloat && bias->numel() == w.size(0)));
  TORCH_CHECK(!logits_out.has_value() || (logits_out->scalar_type() == at::kFloat && logits_out->is_contiguous() &&
                                          logits_out->numel() == x.size(0) * w.size(0)));
  const c10::cuda::CUDAGuard guard(x.device());
  const int rc = b200_linear_xent_eval(x.data_ptr(), w.data_ptr(), opt_ptr<const float>(bias),
                                       reinterpret_cast<const long long*>(target.data_ptr<int64_t>()),
                                       loss_acc.data_ptr<float>(), opt_ptr<float>(logits_out), static_cast<int>(x.size(0)),
                                       static_cast<int>(x.size(1)), static_cast<int>(w.size(0)), cur_stream());
  if (rc == -2) return false;
  check(rc, "linear_xent_eval");
  return true;
}
void mse(const at::Tensor& pred, const at::Tensor& target, const std::optional<at::Tensor>& dpred, at::Tensor loss_acc,
         double grad_scale) {
  CHECK_CUDA(pred);
  TORCH_CHECK(target.scalar_type() == at::kFloat && target.numel() == pred.numel());
  const c10::cuda::CUDAGuard guard(pred.device());
  const int in32 = pred.scalar_type() == at::kFloat;
  const int out32 = dpred.has_value() && dpred->defined() && dpred->scalar_type() == at::kFloat;
  check(b200_mse(pred.data_ptr(), in32, target.data_ptr<float>(), opt_ptr<void>(dpred), out32,
                 loss_acc.data_ptr<float>(), pred.numel(), static_cast<float>(grad_scale), cur_stream()),
        "mse");
}

}  // namespace

PYBIND11_MODULE(TORCH_EXTENSION_NAME, m) {
  m.doc() = "baton_b200 sm_90a kernels";
  m.attr("MAX_RANKS") = B200_MAX_RANKS;
  m.def("gemm", &gemm);
  m.def("trace_set", &trace_set);
  m.def("attention_fwd", &attention_fwd);
  m.def("attention_bwd", &attention_bwd);
  m.def("bn_bwd_cluster", &bn_bwd_cluster);
  m.def("im2col_tma_probe", &im2col_tma_probe);
  m.def("conv_igemm_fwd", &conv_igemm_fwd);
  m.def("conv_igemm_wgrad", &conv_igemm_wgrad);
  m.def("conv_igemm_dgrad", &conv_igemm_dgrad);
  m.def("conv_igemm_dgrad_s2", &conv_igemm_dgrad_s2);
  m.def("conv_halo", &conv_halo);
  m.def("gemm_batched", &gemm_batched);
  m.def("gemm_fp8", &gemm_fp8);
  m.def("quant_mx_rows", &quant_mx_rows);
  m.def("quant_mx_cols", &quant_mx_cols);
  m.def("dequant_mx", &dequant_mx);
  m.def("fused_sgd", &fused_sgd);
  m.def("fused_sgd_segments", &fused_sgd_segments);
  m.def("weighted_sum", &weighted_sum);
  m.def("fold_client", &fold_client);
  m.def("scaffold_corr", &scaffold_corr);
  m.def("scaffold_dc", &scaffold_dc);
  m.def("cast", &cast);
  m.def("gather_rows", &gather_rows);
  m.def("colsum", &colsum);
  m.def("add_bf16", &add_bf16);
  m.def("relu_bwd", &relu_bwd);
  m.def("gelu", &gelu);
  m.def("gelu_bwd", &gelu_bwd);
  m.def("pad_rows", &pad_rows);
  m.def("embedding_bwd", &embedding_bwd);
  m.def("fedavg_allreduce", &fedavg_allreduce);
  m.def("fedavg_allreduce_robust", &fedavg_allreduce_robust);
  m.def("pack_client", &pack_client);
  m.attr("MAX_ROBUST_CLIENTS") = B200_MAX_ROBUST_CLIENTS;
  m.def("flag_barrier", &flag_barrier);
  m.attr("DP_WORK_WORDS") = B200_DP_WORK_WORDS;
  m.def("dp_clip_factor", &dp_clip_factor);
  m.def("fold_client_scaled", &fold_client_scaled);
  m.def("im2col", &im2col);
  m.def("col2im", &col2im);
  m.def("maxpool", &maxpool);
  m.def("maxpool_bwd", &maxpool_bwd);
  m.def("avgpool", &avgpool);
  m.def("avgpool_bwd", &avgpool_bwd);
  m.def("bn_stats", &bn_stats);
  m.def("bn_apply", &bn_apply);
  m.def("bn_bwd_reduce", &bn_bwd_reduce);
  m.def("bn_bwd_apply", &bn_bwd_apply);
  m.def("bn_relu_maxpool", &bn_relu_maxpool);
  m.def("bn_maxpool_bwd", &bn_maxpool_bwd);
  m.def("layernorm_fwd", &layernorm_fwd);
  m.def("layernorm_bwd", &layernorm_bwd);
  m.def("softmax_fwd", &softmax_fwd);
  m.def("softmax_bwd", &softmax_bwd);
  m.def("softmax_xent", &softmax_xent);
  m.def("mse", &mse);
  m.def("linear_xent_head", &linear_xent_head);
  m.def("linear_xent_eval", &linear_xent_eval);
  m.def("bn_fold_eval", &bn_fold_eval);
}
