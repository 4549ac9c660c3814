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

// LoRA term of a bf16 GEMM (b200_gemm_bf16_lora, csrc/lora.cu): D = act(alpha * (A B^T + s T) + bias) with
//     T[m, n] = sum_{j < rs} U[m, t rs + j] * F(t ds + n - sl ds, j),   sl = n / ds, t = slot[sl] (-1: T = 0),
// F(row, j) = f[row * fs_n + j * fs_j].  The forward passes U = X A^T and F = the stacked B of the targeted slices
// (fs_n = rs, fs_j = 1); the data gradient U = V = dY' B and F = A^T (one slice, rs = R, fs_n = 1, fs_j = K).
// R = columns of U in use (multiple of 8, <= B200_LORA_MAX_R), ldu % 8 == 0, U 16-byte aligned, ds % 32 == 0,
// N <= 3 ds; -3 otherwise.
#define B200_LORA_MAX_R 192
struct B200LoraEpilogue {
  const void* u;                    // bf16 [M, ldu]
  long long ldu;
  const void* f;                    // bf16 up factor
  long long fs_n, fs_j;
  int R, rs, ds;
  int slot[3];
  float s;
};
int b200_gemm_bf16_lora(const void* a, const void* b, void* d, const float* bias, int M, int N, int K, long long lda,
                        long long ldb, long long ldd, int a_mn, int b_mn, int out_fp32, int act, float alpha,
                        const B200LoraEpilogue* lora, cudaStream_t stream);
// LoRA down projection (csrc/lora.cu): for each of the T <= 3 slices t and j < rs, k over [0, kt)
//     U[m, t rs + j] = bf16( sum_k X[m, xoff[t] + k] * W[t w_ts + j wsj + k wsk] )      (fp32 accumulation, k ascending)
// forward: T = 1, W = A [R, K] (wsj = K, wsk = 1); backward V = dY' B: xoff[t] = the slice's first column, kt = its width,
// W = the stacked B [T ds, r] (w_ts = ds r, wsj = 1, wsk = r).  rs % 8 == 0, T rs <= B200_LORA_MAX_R.
int b200_lora_down(const void* x, long long ldx, const void* w, long long w_ts, long long wsj, long long wsk, void* u,
                   long long ldu, int M, int T, int rs, int kt, const long long* xoff, cudaStream_t stream);
// LoRA adapter gradient (csrc/lora.cu): for each slice t < T, a < NA, b < NB
//     out[t out_ts + a osa + b osb] += s * sum_m L[m, lo[t] + a] * Q[m, qo[t] + b]
// over M in a fixed split of B200_LORA_SPLIT_ROWS rows per partial (work: T * ceil(M / rows) * NA * NB floats), the
// partials summed in split order by a second kernel: the bits depend on the shapes only.
#define B200_LORA_SPLIT_ROWS 256
int b200_lora_grad(const void* l, long long ldl, const void* q, long long ldq, float* out, long long osa, long long osb,
                   long long out_ts, int M, int NA, int NB, int T, const long long* lo, const long long* qo, float s,
                   float* work, cudaStream_t stream);

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
// the same with dropout on the probabilities (struct B200Dropout below; element i = the index into probs): the
// forward's probs stay the undropped P, out = (P o M s) V; the backward regenerates the mask
struct B200Dropout;
int b200_attention_drop_fwd(const void* qkv, void* out, void* probs, int B, int S, int H, int dh, float scale,
                            const B200Dropout* drop, cudaStream_t stream);
int b200_attention_drop_bwd(const void* qkv, const void* dout, const void* probs, void* dqkv, int B, int S, int H, int dh,
                            float scale, const B200Dropout* drop, cudaStream_t stream);
// the same tiles at 0 < S < 128 (ViT: patches + class token), d_head = 64, no mask or dropout; probs is
// [B*H, S, round_up(S, 8)] with the pad columns written as 0, and no row >= S of out / dqkv is written
int b200_attention_short_fwd(const void* qkv, void* out, void* probs, int B, int S, int H, int dh, float scale,
                             cudaStream_t stream);
int b200_attention_short_bwd(const void* qkv, const void* dout, const void* probs, void* dqkv, int B, int S, int H, int dh,
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
// ---- conv_halo.cu: 3x3 pad-1 convolution, halo-tiled, over a gathered tensor of C = 64 or 128 channels (stride 1) or
// C = 64 (stride 2, forward only); dgrad != 0: input gradient
int b200_conv_halo(const void* src, const void* w, void* out, int N, int H, int W, int C, int Nout, int stride,
                   int dgrad, int mc, float* col_stats, cudaStream_t stream);
// the same kernel from whole small images in shared memory (no halo), bn = 32 or 64 output columns per CTA, over
// C = 256 (stride 1) or C = 128 (stride 2, forward only) gathered channels
int b200_conv_smallmap(const void* src, const void* w, void* out, int N, int H, int W, int C, int Nout, int stride,
                       int dgrad, int mc, int bn, float* col_stats, cudaStream_t stream);
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
                   const float* corr, float* adam_v, int clip, cudaStream_t stream);
// the same step over a device table of n_seg arena chunks {offset, length, kind} (int64 [n_seg][3]); kind 0: with a
// gradient (zeroed afterwards), kind 1: gradient identically zero (never read)
int b200_fused_sgd_segments(float* w, float* g, float* mom, void* w_bf16, const long long* segments, int n_seg,
                            const float* hyper, int nesterov, const float* prox_anchor, const float* corr,
                            float* adam_v, int clip, cudaStream_t stream);
// Gradient-norm clipping (clip_grad_norm_): norm_out[0] = ||g[0, n)|| (fp32; accumulated in fp64 with a fixed grid and
// summation order) and coef_out[0] = min(max_norm[0] / (norm + 1e-6), 1) as torch rounds it.  work: int64
// [B200_GRAD_NORM_WORK_WORDS], zero on first use (partials, arrival counter, fp64 sum of squares); g 16-byte aligned.
// clip != 0 in the two calls above selects their clipped forms, which multiply g by hyper[5] (SGD: hyper is then
// float[6]) or by row[9] (AdamW) as they load it.
#define B200_GRAD_NORM_BLOCKS 528
#define B200_GRAD_NORM_WORK_WORDS (B200_GRAD_NORM_BLOCKS + 2)
int b200_grad_norm_clip(const float* g, long long n, const float* max_norm, void* work, float* norm_out,
                        float* coef_out, cudaStream_t stream);
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
// dst[s] = random crop (zero padding `pad`) + horizontal flip of the NHWC image src[idx[s]], s in [0, n_rows); the
// draws of output position s0 + s come from Philox4x32-10 under `key` with counter (s0 + s, words[0..2]) where words =
// {epoch, stream_lo, stream_hi} is read on the device.  elem_bytes 2 or 4; one image row at most 48 KB
int b200_gather_augment(const void* src, const long long* idx, void* dst, const unsigned* words, long long n_rows,
                        long long s0, unsigned long long key, int pad, int crop, int flip, int H, int W, int C,
                        int elem_bytes, cudaStream_t stream);
// gather_augment, then each image mixed with its batch partner: within every batch of `batch` positions (the last one
// may be shorter), position j pairs with j - 1 (the first with the last); both are augmented with their own draws, then
// mixed under the batch's mix row rows[(s0 + s) / batch] (8 int32: lam, lam1 as fp32 bits, kind 0 mixup / 1 CutMix,
// box y0, y1, x0, x1).  s0 % batch == 0.  elem_bytes 2 (fp16 = 1 for half, else bf16) or 4 (fp32)
int b200_gather_mix(const void* src, const long long* idx, void* dst, const unsigned* words, const int* rows,
                    long long n_rows, long long s0, int batch, unsigned long long key, int pad, int crop, int flip,
                    int H, int W, int C, int elem_bytes, int fp16, cudaStream_t stream);
int b200_colsum(const void* x, float* out, long long rows, int cols, int accumulate, cudaStream_t stream);
int b200_add_bf16(const void* a, const void* b, void* out, long long n, int relu, cudaStream_t stream);
int b200_relu_bwd_bf16(const void* y, const void* dy, void* dx, long long n, cudaStream_t stream);
int b200_gelu_bf16(const void* x, void* y, long long n, cudaStream_t stream);
int b200_gelu_bwd_bf16(const void* x, const void* dy, void* dx, long long n, cudaStream_t stream);
int b200_gelu_erf_bf16(const void* x, void* y, long long n, cudaStream_t stream);
int b200_gelu_erf_bwd_bf16(const void* x, const void* dy, void* dx, long long n, cudaStream_t stream);
int b200_vit_tokens_fwd(const void* z, const float* cls, const float* bias, const float* pos, void* tok, int B, int S,
                        int D, cudaStream_t stream);
int b200_vit_tokens_bwd(const void* dtok, void* dz, float* dcls, float* dbias, float* dpos, int B, int S, int D,
                        cudaStream_t stream);
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
// Every other kind of round has its own args struct derived from FedAvgArgs (FedAvgArgs itself: the plain weighted mean).
// The struct is the kernel's parameter layout and selects the kernel: see b200_fedavg_round below.
// DP-FedAvg round (delta mode, peer loads): clipped weights w_k = n_k s_k / N and Gaussian noise on the reduced sum.
struct FedAvgDPArgs : FedAvgArgs {
  const float* clip_page[B200_MAX_RANKS];   // peer-mapped: clip_page[k][0] = s_k of rank k for this round
  float noise_std;                  // sigma * C (noise on the sum; the kernel divides by N with the weights)
  unsigned long long seed;          // Philox key
  uint32_t round;                   // Philox counter word 2: the collective's round index
};
// SCAFFOLD round (delta mode, peer loads): the plain round over segment 0 plus, between the same two barriers, a second
// segment of n_c elements at byte offset seg1_off of every wire half: each participant (n_k != 0) packs cast(dc), the
// tile owner reduces with weight inv_clients = 1 / N, and every live rank applies c += result.
struct FedAvgScaffoldArgs : FedAvgArgs {
  const float* dc;                  // local: this rank's summed control-variate updates [n_c]
  float* c;                         // local: the server control variate [n_c]
  long long n_c;                    // elements of segment 1 (the parameters; multiple of 8)
  long long seg1_off;               // byte offset of segment 1 inside each wire half (multiple of 16)
  float inv_clients;                // 1 / N, N = the client population
};
// Robust round (delta mode, peer loads, no arrival flags): coordinate-wise median or trimmed mean over the participating
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
// Multi-Krum round (as the robust round: delta mode, peer loads, no arrival flags): the robust round's segments and
// apply, with a selection of whole clients in phase 1.  Every CTA adds the pair sums (x_i - x_j)^2 of its tiles into work[cta][pair]; the last CTA
// of the rank (counter sync[0], zeroed by the launcher) adds them in CTA order into this rank's page dist_page[rank]
// and raises sync[1]; after a per-CTA barrier at epoch + 2 every CTA adds the live ranks' pages in rank order, scores
// every client by the krum_k[P] smallest distances (fp64, ascending), keeps the krum_m[P] lowest (score, position)
// and runs the robust selection over the kept segments with kind = 1 (trimmed mean) and trim_b = 0.  Barrier 2 takes
// epoch + 3, so a launch owns epoch+1 .. epoch+3 as every round does.  CTA 0 writes report: [0] = P, [1 + 32 i + j] =
// D[i][j], [1 + 1024 + i] = score_i, [1 + 1024 + 32 + i] = 1 if client i is kept.
#define B200_KRUM_PAIRS 496         // 32 * 31 / 2: one page / work slot of fp64 pair sums
#define B200_KRUM_MAX_CTAS 296      // work slots; the launcher clamps the grid to it
#define B200_KRUM_REPORT (1 + B200_MAX_ROBUST_CLIENTS * B200_MAX_ROBUST_CLIENTS + 2 * B200_MAX_ROBUST_CLIENTS)
struct FedAvgKrumArgs : FedAvgRobustArgs {
  double* dist_page[B200_MAX_RANKS];   // peer-mapped: this round's half of rank k's distance page (>= 496 doubles)
  double* work;                     // local: [B200_KRUM_MAX_CTAS][B200_KRUM_PAIRS] per-CTA partial sums
  unsigned int* sync;               // local: [2] arrival counter, done flag
  double* report;                   // local: [B200_KRUM_REPORT] or nullptr
  uint8_t krum_k[B200_MAX_ROBUST_CLIENTS + 1];   // neighbours per score for P = 0 .. 32 (host-computed)
  uint8_t krum_m[B200_MAX_ROBUST_CLIENTS + 1];   // clients kept for P = 0 .. 32
};
// Server-optimizer round (ServerOptArgs<the round's struct>, any kind): the apply phase runs FedAvgM / FedAdagrad /
// FedYogi / FedAdam (parallel/server_opt.py) on the parameter elements [0, n_param) instead of global += d, with
// d = decode(wire) * apply_scale:  m = c0*m + d, x += c4*m (kind 0, avgm), or m = c0*m + c1*d, v by kind (1 adagrad:
// v + d*d, 2 yogi: v - c3*(d*d)*sign(v - d*d), 3 adam: c2*v + c3*(d*d)), x += c4*m / (sqrt(v) + c5); every operation
// rounded separately.  c = coef = {b1, 1-b1, b2, 1-b2, lr, tau} in fp32 (host-computed).  Float buffers [n_param, n) keep
// global += d; a round with total weight 0 leaves x, m and v unchanged.  Delta mode only; n_param % 8 == 0.
extern "C++" {
template <class Base>
struct ServerOptArgs : Base {
  float* m;                         // local: first moment over the parameters [n_param]
  float* v;                         // local: second moment [n_param] (nullptr for kind 0)
  long long n_param;                // parameter elements at the start of the arena (multiple of 8)
  int kind;                         // 0 avgm, 1 adagrad, 2 yogi, 3 adam
  float coef[6];                    // b1, 1 - b1, b2, 1 - b2, lr, tau
};
// Personalized round (LocalArgs<FedAvgArgs> or LocalArgs<ServerOptArgs<FedAvgArgs>>: plain weighted mean, no arrival
// flags): the physical arena range [lo, lo + len) holds client-local entries that the round never reads or writes, in
// any buffer.  Base::n is then the LOGICAL element count n_shared = physical n - len; the wire, its tiles, the reduce
// and fp8 block scales work over [0, n_shared) exactly as a plain round over n_shared elements.  The phases that touch the
// replica (pack: theta, global_w; apply: global_w, theta, bf16 shadow, momentum reset, server m / v) address logical
// element e at physical e + (e >= lo ? len : 0).  lo and len are multiples of 1024, so no wire vector or fp8 block
// crosses an edge of the range; n_momentum and the server optimizer's n_param stay physical.
template <class Base>
struct LocalArgs : Base {
  long long lo;                     // first physical element of the local range (multiple of 1024)
  long long len;                    // elements in the local range (multiple of 1024)
};
// One FedAvg round of the kind Args names: FedAvgArgs, FedAvgDPArgs, FedAvgScaffoldArgs, FedAvgRobustArgs,
// FedAvgKrumArgs, FedAvgTopkArgs, FedAvgSecAggArgs (declared below), ServerOptArgs<one of them>, or
// LocalArgs<FedAvgArgs / ServerOptArgs<FedAvgArgs>>.
// Runs fedavg_round_kernel<WIRE, Args> (csrc/fedavg.cu)
// cooperatively on at most n_ctas CTAs; -2 when the arguments do not fit the kind.
template <class Args>
int b200_fedavg_round(const Args* args, int n_ctas, cudaStream_t stream);
}
// one logical client's upload: seg = cast(theta - global_w) in wire format wire_kind (fp8: scales behind the n payload
// bytes), exactly the collective's own pack; reset != 0 also returns the replica to the global model (theta, bf16
// shadow, momentum [0, n_mom)) as b200_fold_client does.  n % 8 == 0, 16-byte aligned fp32 arrays.
int b200_pack_client(void* seg, float* theta, const float* global_w, void* w_bf16, float* mom, long long n_mom,
                     long long n, int wire_kind, int reset, cudaStream_t stream);
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
// Top-k round (fp32 / bf16 wire, delta mode, peer loads, no arrival flags, prepacked): every participant's upload is a
// sparse list in its wire half, written before the launch by b200_topk_pack / b200_nonzero_pack (compress.cu): uint32 rowptr[n / 1024 + 1] at rowptr_off, uint16 off[cap] at off_off (the offset of
// an entry inside its 1024-element granule), values[cap] in the wire dtype at val_off, entries in index order.  The
// owner of a tile adds w_k * value into an fp32 shared-memory tile, live ranks in order (fmaf from 0, skipping w_k == 0,
// as the dense reduce), and stores the cast dense result into seg 0 of every live replica; pack phase: none; barriers,
// apply, loss and integer arena: the plain round's.  n and tile_elems are multiples of 1024.
struct FedAvgTopkArgs : FedAvgArgs {
  long long rowptr_off;             // byte offsets inside every rank's wire half
  long long off_off;
  long long val_off;
};

// Secure-aggregation round (parallel/secagg.py; fp32-sized wire, delta mode, peer loads, no arrival flags, not prepacked):
// a count barrier at epoch + 1 (payload n_k) fixes the participants (live ranks with n_k > 0) and the weights
// w_k = n_k * (1 / N) before the pack; each participant packs u = encode(theta - global) + its pairwise ChaCha20 masks
// (csrc/secagg.cuh) as uint32, 4 per 16 B; barrier at epoch + 2; the owner of a tile adds the participants' u as
// uint32 with wrap-around (the masks cancel) and stores the sum into every live replica; barrier at epoch + 3; the apply
// phase adds fp32(int32(sum)) * 2^-f (or takes the server step on it).  Loss and integer arena: as in the plain round.
struct FedAvgSecAggArgs : FedAvgArgs {
  uint32_t keys[B200_MAX_RANKS][8]; // keys[j]: the ChaCha20 key this rank shares with rank j (unused for j == rank)
  float range;                      // R: the clamp of every update element
  int frac_bits;                    // f = 30 - ceil(log2 R)
  float two_f, inv_two_f;           // 2^f, 2^-f
  unsigned long long* saturated;    // local device counter: elements this rank clamped (or found non-finite)
};
#define B200_SECAGG_MAX_ELEMS (1ll << 36)   // the 32-bit block counter e / 16
// Standalone encode + mask (the pack of a secure round, for NcclSession and tests): out[e] = encode(theta[e] - global_w[e])
// + sum over the n_peers peers of sign[p] * S(keys[p], block counter0 + e / 16, nonce)  (mod 2^32), e in [0, n);
// *saturated += the clamped / non-finite elements.  global_w may be nullptr (x = theta).
struct B200SecAggPeers {
  uint32_t key[B200_MAX_RANKS][8];
  int sign[B200_MAX_RANKS];         // +1 or -1
  int n;
};
int b200_secagg_encode(const float* theta, const float* global_w, long long n, float w, float range, int frac_bits,
                       const B200SecAggPeers* peers, const uint32_t* nonce, uint32_t counter0, uint32_t* out,
                       unsigned long long* saturated, cudaStream_t stream);

// ---- compress.cu: top-k selection with error feedback (parallel/compress.py)
// work: int32 [B200_TOPK_WORK_WORDS(n)] scratch; n % 1024 == 0, 1 <= k <= n, 16-byte aligned fp32 arrays.
#define B200_TOPK_WORK_WORDS(n) (4624 + 4 * ((n) / 1024) + 1)
// u = (theta - global_w) [+ u when ef] (each operation rounded), the k largest |u| (ties: lower index) compacted into
// rowptr / off / val (wire_kind 0 fp32, 1 bf16; cap >= k entries); ef: u = 0 on the kept entries (u is the residual)
int b200_topk_pack(const float* theta, const float* global_w, float* u, int ef, long long n, long long k, int* work,
                   uint32_t* rowptr, uint16_t* off, void* val, int wire_kind, long long cap, cudaStream_t stream);
// the same selection folded into acc: acc (+)= nk * topk(u) (first: from 0), residual as above; reset: theta = global,
// bf16 shadow, momentum [0, n_mom) = 0 (the next co-resident client starts from the global model)
int b200_topk_fold(float* theta, const float* global_w, float* u, int ef, long long n, long long k, int* work, float* acc,
                   float nk, int first, void* w_bf16, float* mom, long long n_mom, int reset, cudaStream_t stream);
// the entries where theta != global_w, value cast(theta - global_w), in the same format (at most cap; the rest dropped)
int b200_nonzero_pack(const float* theta, const float* global_w, long long n, int* work, uint32_t* rowptr, uint16_t* off,
                      void* val, int wire_kind, long long cap, cudaStream_t stream);

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
// GroupNorm over NHWC bf16 [N, HW, C], G groups of C / G channels (csrc/norm.cu).  Forward: y = relu?(gamma * (z -
// mean) * rstd + beta + residual?), mean / rstd fp32 [N, G]; `work` (or nullptr): the backward's buffer, whose G
// counters it zeroes.  Backward: dz, dres = dy' (or nullptr), dgamma / dbeta ACCUMULATED (fixed summation order);
// work: fp32 [G + 2 N C], first G words zero.  Both return -2 when G does not divide C.
int b200_gn_fwd(const void* z, const void* residual, void* y, const float* gamma, const float* beta, float* mean,
                float* rstd, float* work, long long N, long long HW, int C, int G, float eps, int relu, cudaStream_t stream);
int b200_gn_bwd(const void* z, const void* y, const void* dy_a, const void* dy_b, void* dz, void* dres, const float* gamma,
                const float* mean, const float* rstd, float* dgamma, float* dbeta, float* work, long long N, long long HW,
                int C, int G, int relu, cudaStream_t stream);
// eval-mode BatchNorm folding: one block per BatchNorm; table = int64 [n_bn][7] {gamma, beta, running_mean,
// running_var (element offsets into arena; gamma / beta -1 = none), output offset, C, eps as float bits}
int b200_bn_fold_eval(const float* arena, const long long* table, int n_bn, float* out, cudaStream_t stream);
int b200_layernorm_fwd(const void* x, const void* residual, void* y, const float* gamma, const float* beta,
                       float* mean, float* rstd, long long rows, int C, float eps, cudaStream_t stream);
int b200_layernorm_bwd(const void* x, const void* dy, void* dx, const float* gamma, const float* mean,
                       const float* rstd, float* dgamma, float* dbeta, long long rows, int C, cudaStream_t stream);
int b200_layernorm_sum_fwd(const void* x, const void* residual, void* y, void* sum, const float* gamma,
                           const float* beta, float* mean, float* rstd, long long rows, int C, float eps,
                           cudaStream_t stream);
int b200_layernorm_sum_bwd(const void* s, const void* dy, const void* ds, void* dsum, const float* gamma,
                           const float* mean, const float* rstd, float* dgamma, float* dbeta, long long rows, int C,
                           cudaStream_t stream);
int b200_softmax_fwd(const void* x, void* y, long long rows, int C, float scale, cudaStream_t stream);
int b200_softmax_bwd(const void* y, const void* dy, void* dx, long long rows, int C, float scale,
                     cudaStream_t stream);

// ---- dropout.cu (and the dropout forms of the fused attention): the mask of one dropout site (csrc/dropout.cuh,
// baton_b200/data/dropout.py).  words: device int32 {epoch, stream_lo, stream_hi}; the run's local step is
// t = epoch * steps + step.  Element i is kept iff word i & 3 of philox4x32_10((i >> 2, 0x80000000 | site << 22 | t,
// stream_lo, stream_hi), key) >= thresh; a kept value is multiplied by scale.  site < 512, t < 2^22.
struct B200Dropout {
  const int* words;
  unsigned long long key;
  uint32_t site, step, steps;
  uint32_t thresh;                  // floor(p * 2^32)
  float scale;                      // fp32(1 / (1 - p))
};
// LayerNorm with dropout: mode 1 (input dropout) pre = drop(x) + residual?, y = LN(pre) (pre written, bf16); mode 2
// (output dropout) y = drop(LN(x + residual?)).  Backward: x = the pre-norm input; mode 1 writes dx = dpre and
// dxd = M s dpre, mode 2 applies M s to dy as it loads it (dxd unused).  dgamma / dbeta ACCUMULATED.
int b200_layernorm_drop_fwd(const void* x, const void* residual, void* y, void* pre, const float* gamma,
                            const float* beta, float* mean, float* rstd, long long rows, int C, float eps, int mode,
                            const B200Dropout* drop, cudaStream_t stream);
int b200_layernorm_drop_bwd(const void* x, const void* dy, void* dx, void* dxd, const float* gamma, const float* mean,
                            const float* rstd, float* dgamma, float* dbeta, long long rows, int C, int mode,
                            const B200Dropout* drop, cudaStream_t stream);
// softmax with dropout: y = softmax(scale x) (saved), yd = drop(y); backward dx = scale y (g - sum(g y)), g = M s dy
int b200_softmax_drop_fwd(const void* x, void* y, void* yd, long long rows, int C, float scale, const B200Dropout* drop,
                          cudaStream_t stream);
int b200_softmax_drop_bwd(const void* y, const void* dy, void* dx, long long rows, int C, float scale,
                          const B200Dropout* drop, cudaStream_t stream);
// y = drop(x) over n bf16 elements (forward and backward of an elementwise dropout)
int b200_dropout(const void* x, void* y, long long n, const B200Dropout* drop, cudaStream_t stream);

// ---- loss.cu
int b200_softmax_xent(const void* logits, int logits_fp32, const long long* target, void* dlogits, int dl_fp32,
                      float* loss_acc, long long rows, int C, long long ld, float grad_scale, cudaStream_t stream);
// linear classifier head + softmax cross-entropy, forward AND backward, one launch (classes <= 32)
int b200_linear_xent_head(const void* x, const void* w, const float* bias, const long long* target, void* dx, float* dw,
                          float* db, float* loss_acc, float* logits_out, int rows, int K, int NC, float grad_scale,
                          cudaStream_t stream);
// soft-target forms (mixup / CutMix / label smoothing, data/mix.py): target of row r is (1 - eps)(lam 1[target[r]] +
// lam1 1[target[r - 1 mod rows]]) + eps / C with lam, lam1 the fp32 words 0, 1 of mix_row (nullable: lam = 1, lam1 = 0)
int b200_softmax_xent_soft(const void* logits, int logits_fp32, const long long* target, void* dlogits, int dl_fp32,
                           float* loss_acc, long long rows, int C, long long ld, float grad_scale, const int* mix_row,
                           float eps, cudaStream_t stream);
int b200_linear_xent_head_soft(const void* x, const void* w, const float* bias, const long long* target, void* dx,
                               float* dw, float* db, float* loss_acc, int rows, int K, int NC, float grad_scale,
                               const int* mix_row, float eps, cudaStream_t stream);
// forward-only head (evaluation): loss_acc[0] += sum of the row losses, loss_acc[1] += #correct
int b200_linear_xent_eval(const void* x, const void* w, const float* bias, const long long* target, float* loss_acc,
                          float* logits_out, int rows, int K, int NC, cudaStream_t stream);
int b200_mse(const void* pred, int pred_fp32, const float* target, void* dpred, int dp_fp32, float* loss_acc,
             long long n, float grad_scale, cudaStream_t stream);
}
