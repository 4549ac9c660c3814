// C launch API of the sm_90a kernels (implemented in the .cu files, wrapped for PyTorch in
// bindings.cpp).  Every launcher takes raw device pointers and a stream and returns 0 or a
// CUDA error code, so the .cu files do not include any PyTorch header and compile in seconds.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#define B200_MAX_RANKS 16

extern "C" {

// Optimizer epilogue of a weight-gradient GEMM: instead of accumulating the gradient into D, apply the SGD step to the
// parameters in place.  theta / theta_bf16 / mom point at the element that D[0, 0] would address and are indexed like
// D (same ldd).  hyper = device float[4] as for b200_fused_sgd (float[5] with an anchor).  A launcher that cannot apply
// it returns B200_SGD_EPILOGUE_DECLINED and touches nothing; the caller then accumulates the gradient as usual.
struct B200SgdEpilogue {
  float* theta;
  void* theta_bf16;                 // or nullptr
  float* mom;                       // or nullptr (no momentum buffer)
  const float* hyper;
  int nesterov;
  const float* anchor;              // FedProx anchor (global model), indexed like theta, or nullptr (no proximal term)
  const float* corr;                // SCAFFOLD correction c - c_i, indexed like theta, or nullptr (exclusive with anchor)
  float* v;                         // AdamW second moment, indexed like theta, or nullptr (SGD).  With it, mom is the
                                    // first moment and hyper the step's AdamW row (ADAMW_ROW floats, csrc/sgd.cuh)
};
#define B200_SGD_EPILOGUE_DECLINED (-6)

// Eval-mode BatchNorm epilogue of a forward convolution GEMM: D = relu?(acc * scale[c] + shift[c] + residual[r, c]) in
// bf16, with the per-column scale / shift that bn_fold_eval derives from the running statistics.  residual is optional
// (bf16, row pitch ldr).  Needs N % 8 == 0, 16-byte aligned scale / shift / residual and ldr % 8 == 0.  A launcher that
// cannot apply it returns B200_AFFINE_EPILOGUE_DECLINED and touches nothing; the caller then runs the GEMM and bn_apply.
struct B200AffineEpilogue {
  const float* scale;
  const float* shift;
  const void* residual;             // or nullptr
  long long ldr;
  int relu;
};
#define B200_AFFINE_EPILOGUE_DECLINED (-7)

// ---- gemm_wgmma.cu
// sgd != nullptr: optimizer epilogue (accumulate, fp32 D, MN-major operands, single K pass on the fixed-depth kernel)
// affine != nullptr: eval-mode BatchNorm epilogue (bf16 D, act 0, no bias / split-K partials; fixed or cluster kernel)
int b200_gemm_bf16(const void* a, const void* b, void* d, const float* bias, int M, int N, int K, long long lda,
                   long long ldb, long long ldd, int a_mn, int b_mn, int out_fp32, int act, int split_k, int accumulate,
                   float alpha, const uint32_t* tile_flags, uint32_t flag_epoch, long long flag_elem_off, int flag_tile_elems,
                   long long flag_bias_off, int force_bn, float* col_stats, const uint32_t* flag_epoch_ptr,
                   const B200SgdEpilogue* sgd, const B200AffineEpilogue* affine, cudaStream_t stream);
int b200_gemm_bf16_batched(const void* a, const void* b, void* d, int M, int N, int K, long long lda, long long ldb,
                           long long ldd, int a_mn, int b_mn, int out_fp32, int act, float alpha, int n_outer,
                           int n_inner, long long a_outer, long long a_inner, long long b_outer, long long b_inner,
                           long long d_outer, long long d_inner, int accumulate, cudaStream_t stream);
// ---- attention.cu (experimental fused attention forward, S = 128, d_head = 64)
int b200_attention_fwd(const void* qkv, void* out, void* probs, int B, int S, int H, int dh, float scale,
                       cudaStream_t stream);
int b200_attention_bwd(const void* qkv, const void* dout, const void* probs, void* dqkv, int B, int S, int H, int dh,
                       float scale, cudaStream_t stream);
// ---- implicit-GEMM convolution (experimental: gemm_wgmma.cu CONV modes fed by TMA im2col maps)
int b200_conv_igemm_fwd(const void* x, const void* w, void* y, int N, int H, int W, int Cin, int Cout, int KH, int KW,
                        int stride, int pad, int Ho, int Wo, int cluster_k, int force_bn, float* col_stats,
                        const B200AffineEpilogue* affine, cudaStream_t stream);
int b200_conv_igemm_dgrad(const void* dy, const void* w, void* dx, int N, int H, int W, int Cin, int Cout, int KH, int KW,
                          int pad, int Ho, int Wo, int cluster_k, int force_bn, cudaStream_t stream);
int b200_conv_igemm_dgrad_s2(const void* dy, const void* w, void* dx, int N, int H, int W, int Cin, int Cout, int KH,
                             int KW, int Ho, int Wo, const int* ntaps, const int* taps, int force_bn, cudaStream_t stream);
int b200_conv_igemm_wgrad(const void* dy, const void* x, float* dw, int N, int H, int W, int Cin, int Cout, int KH, int KW,
                          int stride, int pad, int Ho, int Wo, int split_k, int force_bn, const B200SgdEpilogue* sgd,
                          cudaStream_t stream);
// ---- conv_halo.cu: 3x3 stride-1 pad-1 convolution over one 64-channel block, halo-tiled (dgrad != 0: input gradient)
int b200_conv_halo(const void* src, const void* w, void* out, int N, int H, int W, int Nout, int dgrad, int mc,
                   float* col_stats, cudaStream_t stream);
// ---- im2col_tma.cu (experimental: TMA im2col tensor maps, probe kernel only)
int b200_im2col_tma_probe(const void* x, void* col, int N, int H, int W, int C, int KH, int KW, int stride, int pad,
                          int Ho, int Wo, cudaStream_t stream);
// ---- gemm_fp8.cu / quant.cu (MXFP8: e4m3 + UE8M0 scale per 32 elements of K)
int b200_gemm_fp8(const void* a, const void* b, void* d, const float* bias, const void* sfa, const void* sfb, int M, int N,
                  int K, long long lda, long long ldb, long long ldd, int out_fp32, int act, int split_k, int accumulate,
                  float alpha, cudaStream_t stream);
int b200_quant_mx_rows(const void* x, void* q, void* sf, long long R, int C, long long ld_in, int Cp, cudaStream_t stream);
int b200_quant_mx_cols(const void* x, void* q, void* sf, long long R, int C, long long ld_in, long long Rp,
                       cudaStream_t stream);
int b200_dequant_mx(const void* q, const void* sf, float* out, long long R, int C, int Cp, cudaStream_t stream);
int b200_gemm_simt(const void* a, const void* b, void* d, const float* bias, int M, int N, int K, long long lda,
                   long long ldb, long long ldd, int a_mn, int b_mn, int out_fp32, int act, int accumulate,
                   float alpha, cudaStream_t stream);

// ---- elementwise.cu
// hyper = device float[4] {lr, momentum, weight_decay, dampening}; with prox_anchor != nullptr float[5], the fifth being
// the FedProx coefficient mu of the term mu * (w - prox_anchor) added to the gradient (prox_anchor indexed like w)
// corr != nullptr (SCAFFOLD, exclusive with prox_anchor): the correction c - c_i, indexed like w, added to the gradient
// wire_slot != nullptr: also emit the client's wire copy for the round-end collective (see SgdPack in elementwise.cu)
// adam_v != nullptr: the AdamW step instead of SGD (no anchor, no correction): mom is the first moment, adam_v the
// second, hyper the step's AdamW row of ADAMW_ROW floats (csrc/sgd.cuh); nesterov is not read
int b200_fused_sgd(float* w, float* g, float* mom, void* w_bf16, long long n, const float* hyper, int zero_grad,
                   int nesterov, const unsigned long long* wire_slot, const float* pack_global,
                   const float* pack_scale, long long n_pack, int wire_fp32, const float* prox_anchor,
                   const float* corr, float* adam_v, cudaStream_t stream);
// the same step over a device table of n_seg arena chunks {offset, length, kind} (int64 [n_seg][3]); kind 0: with a
// gradient (zeroed afterwards), kind 1: gradient identically zero (never read)
int b200_fused_sgd_segments(float* w, float* g, float* mom, void* w_bf16, const long long* segments, int n_seg,
                            const float* hyper, int nesterov, const float* prox_anchor, const float* corr,
                            float* adam_v, cudaStream_t stream);
// SCAFFOLD control variates over n parameters (n % 4 == 0, 16-byte aligned): corr = c - c_i before a client trains;
// after it trained, dc = (global_w - theta) * inv_k_eta - c, c_i += dc, up = dc (first != 0) or up += dc
int b200_scaffold_corr(float* corr, const float* c, const float* ci, long long n, cudaStream_t stream);
int b200_scaffold_dc(float* up, float* ci, const float* c, const float* global_w, const float* theta, long long n,
                     float inv_k_eta, int first, cudaStream_t stream);
// logical-client fold: acc (+)= nk * (theta - global) [+ reset of the replica]; mode 2: theta = global + acc * nk
int b200_fold_client(float* acc, float* theta, const float* global_w, void* w_bf16, float* mom, long long n_mom, long long n,
                     float nk, int mode, int reset, cudaStream_t stream);
int b200_weighted_sum(void* dst, const void* const* srcs, const float* weights, int n_src, long long n, int dtype,
                      cudaStream_t stream);  // dtype: 0 fp32, 1 bf16
int b200_cast_f32_bf16(const float* src, void* dst, long long n, cudaStream_t stream);
int b200_cast_bf16_f32(const void* src, float* dst, long long n, cudaStream_t stream);
int b200_gather_rows(const void* src, const long long* idx, void* dst, long long n_rows, long long row_bytes,
                     cudaStream_t stream);
int b200_gather_rows_i64(const long long* src, const long long* idx, long long* dst, long long n,
                         cudaStream_t stream);
int b200_colsum(const void* x, float* out, long long rows, int cols, int accumulate, cudaStream_t stream);
int b200_add_bf16(const void* a, const void* b, void* out, long long n, int relu, cudaStream_t stream);
int b200_relu_bwd_bf16(const void* y, const void* dy, void* dx, long long n, cudaStream_t stream);
int b200_gelu_bf16(const void* x, void* y, long long n, cudaStream_t stream);
int b200_gelu_bwd_bf16(const void* x, const void* dy, void* dx, long long n, cudaStream_t stream);
int b200_embedding_bwd(const void* dy, const long long* idx, float* grad, long long n_rows, int width,
                       cudaStream_t stream);
// flags != nullptr: wait (bounded) until the arrival flags covering arena elements [elem_off, elem_off + rows * k) have
// reached *epoch_word before reading src (bcast_gemm staging of a weight whose K is not TMA-aligned)
int b200_pad_rows_bf16(const void* src, void* dst, long long rows, int k, int kp, const uint32_t* flags,
                       const uint32_t* epoch_word, long long elem_off, int granule, cudaStream_t stream);

// ---- fedavg.cu
struct FedAvgArgs {
  void* wire[B200_MAX_RANKS];       // peer-mapped wire buffers (index = rank); wire[rank] is local
  unsigned long long* pads[B200_MAX_RANKS];  // peer-mapped 64-bit barrier pads: (epoch << 32) | payload
  void* wire_mc;                    // multicast address of the wire buffer (NVLS) or nullptr
  float* theta;                     // local fp32 master weights [n]
  float* global_w;                  // local fp32 copy of the global model [n] (needed in delta mode)
  void* theta_bf16;                 // local bf16 shadow weights [n] or nullptr
  float* momentum;                  // optional: momentum buffer [n_momentum] reset when the round ends
  long long n_momentum;
  long long* int_local;             // local int64 side arena (num_batches_tracked ...) or nullptr
  long long* int_wire[B200_MAX_RANKS];  // peer-mapped copies of the int side arena
  float* loss_local;                // local per-epoch losses [n_loss] or nullptr
  float* loss_wire[B200_MAX_RANKS]; // peer-mapped per-epoch loss pages
  float* loss_out;                  // local: sample-weighted per-epoch loss of the round [n_loss]
  int n_loss;
  float n_samples[B200_MAX_RANKS];  // n_k per rank (0 = not a participant); [rank] is always valid
  int counts_from_flags;            // 1: peers' n_k ride on the barrier flags (no host exchange)
  float nvls_prescale;              // NVLS: wire = n_k * prescale * x, applied as sum / (N * prescale)
  uint32_t alive_mask;              // ranks that take part in the collective (readers / receivers)
  int rank, world;
  long long n;                      // float elements in the arena
  int n_int;
  int wire_kind;                    // 0: fp32 wire, 1: bf16, 2: block-scaled fp8 (e4m3 + UE8M0 / 32)
  int delta;                        // 1: upload theta - global, result applied as global += sum
  int use_nvls;                     // 1: multimem.ld_reduce / multimem.st on wire_mc
  uint32_t epoch;                   // barrier epoch base (this launch uses epoch+1 .. epoch+3)
  uint32_t* tile_flags;             // optional local per-tile arrival flags (bcast_gemm) or nullptr
  uint32_t flag_value;              // value published into tile_flags
  int tile_elems;                   // arena tile size in elements
  int prepacked;                    // 1: the wire already holds this round's upload (emitted by the last SGD step): skip phase 0
  int timeout_log2;                 // spin limit (2^k polls) before the kernel gives up, 0 = none
  int* status;                      // device int: set non-zero on barrier timeout
  unsigned long long* phase_ns;     // optional [16]: %globaltimer at the phase boundaries (first / last CTA), or nullptr
};
// DP-FedAvg round (fedavg_allreduce_kernel<WIRE, true>): clipped weights w_k = n_k s_k / N and Gaussian noise on the
// reduced sum.  A separate type derived from FedAvgArgs, so the plain kernels and flag_barrier_kernel keep their
// parameter layout.
struct FedAvgDPArgs : FedAvgArgs {
  const float* clip_page[B200_MAX_RANKS];   // peer-mapped: clip_page[k][0] = s_k of rank k for this round
  float noise_std;                  // sigma * C (noise on the sum; the kernel divides by N with the weights)
  unsigned long long seed;          // Philox key
  uint32_t round;                   // Philox counter word 2: the collective's round index
};
// SCAFFOLD round (fedavg_allreduce_scaffold_kernel<WIRE>): the plain round over segment 0 plus, between the same two
// barriers, a second segment of n_c elements at byte offset seg1_off of every wire half: each participant (n_k != 0)
// packs cast(dc), the tile owner reduces with weight inv_clients = 1 / N, and every live rank applies c += result.
struct FedAvgScaffoldArgs : FedAvgArgs {
  const float* dc;                  // local: this rank's summed control-variate updates [n_c]
  float* c;                         // local: the server control variate [n_c]
  long long n_c;                    // elements of segment 1 (the parameters; multiple of 8)
  long long seg1_off;               // byte offset of segment 1 inside each wire half (multiple of 16)
  float inv_clients;                // 1 / N, N = the client population
};
// Robust round (fedavg_allreduce_robust_kernel<WIRE>): coordinate-wise median or trimmed mean over the participating
// CLIENTS instead of the weighted mean.  Each wire half holds up to S client segments of seg_stride bytes
// ([seg 0 | pad | seg 1 | ...], seg 0 at the half's start = the plain layout); rank k publishes its segment count m_k in
// its page seg_page[k][0] (written by the kernel from my_segs), P = sum of m_k over the live ranks <= 32.  The owner of a
// tile sorts the P decoded values of every element (total order, NaN above +inf), selects, and stores cast(result) into
// seg 0 of every live replica; the apply phase is the plain one.  Loss and integer arena: as in the plain round.
#define B200_MAX_ROBUST_CLIENTS 32
struct FedAvgRobustArgs : FedAvgArgs {
  uint32_t* seg_page[B200_MAX_RANKS];   // peer-mapped: seg_page[k][0] = m_k of rank k for this round
  uint32_t my_segs;                 // m_r of this rank (0: not a participant)
  long long seg_stride;             // bytes from one client segment to the next (multiple of 256)
  int kind;                         // 0: median, 1: trimmed mean
  uint8_t trim_b[B200_MAX_ROBUST_CLIENTS + 1];   // trimmed mean: b = floor(beta * P) for P = 0 .. 32 (host-computed)
};
int b200_fedavg_allreduce(const FedAvgArgs* args, int n_ctas, cudaStream_t stream);
int b200_fedavg_allreduce_robust(const FedAvgRobustArgs* args, int n_ctas, cudaStream_t stream);   // delta, peer loads
// one logical client's upload: seg = cast(theta - global_w) in wire format wire_kind (fp8: scales behind the n payload
// bytes), exactly the collective's own pack; reset != 0 also returns the replica to the global model (theta, bf16
// shadow, momentum [0, n_mom)) as b200_fold_client does.  n % 8 == 0, 16-byte aligned fp32 arrays.
int b200_pack_client(void* seg, float* theta, const float* global_w, void* w_bf16, float* mom, long long n_mom,
                     long long n, int wire_kind, int reset, cudaStream_t stream);
int b200_fedavg_allreduce_dp(const FedAvgDPArgs* args, int n_ctas, cudaStream_t stream);   // delta mode, peer loads only
int b200_fedavg_allreduce_scaffold(const FedAvgScaffoldArgs* args, int n_ctas, cudaStream_t stream);   // delta, peer loads
// DP clip factor: s = min(1, clip / ||theta - global_w||_2) over [0, n), norm in fp64 (s = 0 when it is not finite), written to
// s_out[0] (and s_copy[0] when given), the norm to norm_out[0]; a non-finite norm adds 1 to *nonfinite (optional).
// Deterministic: fixed grid, per-block partials in work (int64 [B200_DP_WORK_WORDS], zero on first use), last-block finish.
#define B200_DP_NORM_BLOCKS 264
#define B200_DP_WORK_WORDS (B200_DP_NORM_BLOCKS + 1)
int b200_dp_clip_factor(const float* theta, const float* global_w, long long n, float clip, void* work, float* s_out,
                        float* norm_out, float* s_copy, int* nonfinite, cudaStream_t stream);
// clipped logical-client fold: acc (+)= s[0] * (theta - global) with s read from device memory, reset as b200_fold_client
int b200_fold_client_scaled(float* acc, float* theta, const float* global_w, void* w_bf16, float* mom, long long n_mom,
                            long long n, const float* s, int first, int reset, cudaStream_t stream);
int b200_flag_barrier(unsigned long long* const* pads, int rank, int world, uint32_t alive_mask, uint32_t epoch,
                      int slot, cudaStream_t stream);

// ---- conv.cu
int b200_im2col_nhwc(const void* x, void* col, int N, int H, int W, int C, int KH, int KW, int stride, int pad,
                     int Ho, int Wo, int kp, cudaStream_t stream);
int b200_col2im_nhwc(const void* col, void* dx, int N, int H, int W, int C, int KH, int KW, int stride, int pad,
                     int Ho, int Wo, int kp, cudaStream_t stream);
int b200_maxpool_nhwc(const void* x, void* y, int* argmax, int N, int H, int W, int C, int k, int stride, int pad,
                      int Ho, int Wo, int arg_u8, cudaStream_t stream);
int b200_maxpool_bwd_nhwc(const void* dy, const void* dy_b, const int* argmax, void* dx, int N, int H, int W, int C, int Ho,
                          int Wo, int k, int stride, int pad, int arg_u8, cudaStream_t stream);
int b200_avgpool_nhwc(const void* x, void* y, int N, int HW, int C, cudaStream_t stream);
int b200_avgpool_bwd_nhwc(const void* dy, void* dx, int N, int HW, int C, cudaStream_t stream);

// ---- norm.cu
int b200_bn_stats(const void* x, float* sums, long long rows, int C, cudaStream_t stream);
int b200_bn_apply(const void* x, const void* residual, void* y, float* sums, const float* gamma, const float* beta,
                  float* running_mean, float* running_var, float* save_mean, float* save_rstd, long long* nbt,
                  long long rows, int C, float eps, float momentum, int relu, int training, cudaStream_t stream);
int b200_bn_bwd_reduce(const void* x, const void* y, const void* dy, const float* save_mean, const float* save_rstd,
                       float* sums, long long rows, int C, int relu, cudaStream_t stream);
int b200_bn_bwd_apply(const void* x, const void* y, const void* dy, void* dx, void* dres, const float* gamma,
                      const float* save_mean, const float* save_rstd, float* sums, float* dgamma, float* dbeta,
                      long long rows, int C, int relu, cudaStream_t stream);
int b200_bn_relu_maxpool(const void* z, void* p, void* argmax, const float* sums, const float* gamma, const float* beta,
                         float* running_mean, float* running_var, float* save_mean, float* save_rstd, long long* nbt, int N,
                         int H, int W, int C, int k, int stride, int pad, int Ho, int Wo, float eps, float momentum,
                         cudaStream_t stream);
int b200_bn_maxpool_bwd(const void* z, const void* p, const void* argmax, const void* dy_a, const void* dy_b, void* dz,
                        const float* gamma, const float* save_mean, const float* save_rstd, float* sums, float* dgamma,
                        float* dbeta, int N, int H, int W, int C, int k, int stride, int pad, int Ho, int Wo,
                        cudaStream_t stream);
int b200_bn_bwd_cluster(const void* x, const void* y, const void* dy_a, const void* dy_b, void* dx, void* dres,
                        const float* gamma, const float* save_mean, const float* save_rstd, float* dgamma, float* dbeta,
                        long long rows, int C, int relu, int max_cluster, cudaStream_t stream);
// eval-mode BatchNorm folding: one block per BatchNorm; table = int64 [n_bn][7] {gamma, beta, running_mean,
// running_var (element offsets into arena; gamma / beta -1 = none), output offset, C, eps as float bits}
int b200_bn_fold_eval(const float* arena, const long long* table, int n_bn, float* out, cudaStream_t stream);
int b200_layernorm_fwd(const void* x, const void* residual, void* y, const float* gamma, const float* beta,
                       float* mean, float* rstd, long long rows, int C, float eps, cudaStream_t stream);
int b200_layernorm_bwd(const void* x, const void* dy, void* dx, const float* gamma, const float* mean,
                       const float* rstd, float* dgamma, float* dbeta, long long rows, int C, cudaStream_t stream);
int b200_softmax_fwd(const void* x, void* y, long long rows, int C, float scale, cudaStream_t stream);
int b200_softmax_bwd(const void* y, const void* dy, void* dx, long long rows, int C, float scale,
                     cudaStream_t stream);

// ---- loss.cu
int b200_softmax_xent(const void* logits, int logits_fp32, const long long* target, void* dlogits, int dl_fp32,
                      float* loss_acc, long long rows, int C, long long ld, float grad_scale, cudaStream_t stream);
// linear classifier head + softmax cross-entropy, forward AND backward, one launch (classes <= 32)
int b200_linear_xent_head(const void* x, const void* w, const float* bias, const long long* target, void* dx, float* dw,
                          float* db, float* loss_acc, float* logits_out, int rows, int K, int NC, float grad_scale,
                          cudaStream_t stream);
// forward-only head (evaluation): loss_acc[0] += sum of the row losses, loss_acc[1] += #correct
int b200_linear_xent_eval(const void* x, const void* w, const float* bias, const long long* target, float* loss_acc,
                          float* logits_out, int rows, int K, int NC, cudaStream_t stream);
int b200_mse(const void* pred, int pred_fp32, const float* target, void* dpred, int dp_fp32, float* loss_acc,
             long long n, float grad_scale, cudaStream_t stream);
}
