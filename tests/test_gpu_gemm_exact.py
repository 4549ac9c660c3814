"""The bf16 GEMM and convolution kernels (csrc/gemm_wgmma.cu, csrc/gemm_simt.cu, csrc/conv_halo.cu) against float64,
at their dispatch branches and edges.  Every case is built on the CPU from a seeded generator.

Family E (exact).  Operands are in {-2, ..., 2}; bias, shift, residual and prefilled accumulators are integers; alpha
and the eval scale are powers of two.  Each case picks a density such that ``max_ij sum_k |a_ik b_kj| <= 2^12``
(asserted).  Every partial sum, in any order, is then an integer below 2^12.  That is exact in fp32 (atomics and the
DSMEM reduce included), and exact even for a k-step that aligned its products to a window as narrow as 13 bits.  So:
* fp32 outputs equal the float64 reference exactly;
* bf16 outputs equal its round-to-nearest-even.  Bf16 cases hold results above 256 (asserted), where the bf16 spacing
  is 2 or more: ties such as 257 -> 256 and 259 -> 260 fail a truncating or ties-away conversion (asserted too);
* fused column statistics (sum and sum of squares of the bf16 output) are exact, because both stay below 2^24
  (asserted);
* tanh-GELU is compared with the float64 GELU of the exact accumulator ``v``: ``|got - ref| <= 2^-19 |v|``.  A bf16
  output must be the correct rounding of a value that close: ``ref`` rounded to nearest-even unless a bf16 midpoint
  lies that close.
Sensitivity: every 16-wide k group of a GEMM, every (tap, 16-channel group) of a convolution and every 16-pixel group
of a weight gradient contributes a nonzero term to some output (asserted with a random projection), so dropping or
repeating one changes the answer.  Hot rows and columns share one sign pattern over part of K, so their products add
up to the results above 256.

Family F (full mantissa).  Operands are ``randn`` rounded to bf16: this catches operands that lose mantissa bits
(values in {-2..2} survive even an e4m3 cast) and intermediates rounded to bf16.
* fp32 outputs: ``rms(got - ref) <= 2^-14 rms(ref)``.  A correct fp32 accumulation at K = 4608 is near 2^-20; one bf16
  rounding of a split-K partial is near 2^-11.
* bf16 outputs: every element is the correct rounding of a value within ``w = 2^-18 sum_k |a_k b_k|`` of ``ref``.  Where
  no bf16 midpoint lies within ``w`` that is ``ref`` rounded to nearest-even; where one does, either neighbour.  An
  element more than one ulp off is accepted only where ``w`` spans several bf16 steps.  This happens for outputs
  thousands of times smaller than the terms summed into them, where the fp32 accumulator's own rounding is larger
  than a bf16 ulp of the result; the H100 shows such elements in every large case.
Each F case prints its ratio, the fraction of elements with a midpoint inside ``w``, and the least pre-rounding error
that explains its worst element that is not correctly rounded (``pytest -rP``).  Measured on one H100 80GB HBM3 at a
700 W power limit:
* fp32 rms ratio: 2^-23.4 to 2^-19.8, and 2^-18.6 for atomic split-K 7 at K = 16384;
* bf16: 4.5 % to 18.8 % of the elements have a midpoint inside ``w``, and the worst implied error is
  2^-22.5 sum|ab| (the stride-1 128-channel halo forward), well inside ``w``.

Every output is written into a view of a larger buffer prefilled with a NaN bit pattern: extra rows after M, a row
pitch ``ldd > N`` for GEMMs, a tail after the last element.  The guard elements must keep their bits, and an output
element the kernel never writes stays NaN and fails the comparison."""
import functools
import math
import re
from collections import namedtuple

import pytest
import torch
import torch.nn.functional as TF

from baton_b200.ops import functional as F

BF16, F32, F64 = torch.bfloat16, torch.float32, torch.float64
EXACT_BOUND = 2 ** 12          # max_ij sum_k |a_ik b_kj| of a family-E case
STATS_BOUND = 2 ** 24          # column sums of squares stay exact in fp32 below this
SENTINEL = {BF16: (torch.int16, 0x7FC1), F32: (torch.int32, 0x7FC00BAD)}     # NaN bit patterns of the guards

Case = namedtuple("Case", "id op geo opts fams kernels")


# ------------------------------------------------------------------------------------------------ the case table
def _g(cid, M, N, K, *, a_mn=False, b_mn=False, bn=0, split_k=1, outs=(F32, BF16), fams="E", kernels=(), **opts):
    return Case(cid, "gemm", dict(M=M, N=N, K=K, a_mn=a_mn, b_mn=b_mn, bn=bn, split_k=split_k),
                dict(outs=outs, **opts), fams, frozenset(kernels))


def _c(cid, op, n, h, w, cin, cout, k, stride, pad, *, fams="E", kernels=(), **opts):
    return Case(cid, op, dict(n=n, h=h, w=w, cin=cin, cout=cout, k=k, stride=stride, pad=pad), opts, fams,
                frozenset(kernels))


def _b(cid, which, B, H, S, dh, *, fams="E", kernels=(), **opts):
    return Case(cid, "batched", dict(which=which, B=B, H=H, S=S, dh=dh), dict(outs=(F32, BF16), **opts), fams,
                frozenset(kernels))


def fixed(bn, stages, conv=0, affine=0):
    return "fixed<{},{},{},{}>".format(bn, stages, conv, affine)


def splitk(bn, conv=0, affine=0, cluster=1):
    return "splitk<{},{},{},{}>".format(bn, cluster, conv, affine)


def persistent(bn, stages):
    return "persistent<{},{}>".format(bn, stages)


SIMT = "simt"


def halo(dgrad, cb, stride):
    return "halo<{},{},{}>".format(int(dgrad), cb, stride)


CASES = [
    # every operand-major combination; BN 64 / 128 with shallow (<= 4 k tiles) and deep rings; ragged M and N, K not a
    # multiple of 64, K < 64
    _g("gemm_kk_bn128_deep", 300, 520, 328, bn=128, fams="EF", kernels=[fixed(128, 6)]),
    _g("gemm_kn_bn64_shallow", 296, 200, 200, b_mn=True, bn=64, kernels=[fixed(64, 4)]),
    _g("gemm_nk_bn128_shallow", 296, 136, 136, a_mn=True, bn=128, kernels=[fixed(128, 3)]),
    _g("gemm_nn_bn64_deep", 264, 72, 1000, a_mn=True, b_mn=True, bn=64, fams="EF", kernels=[fixed(64, 8)]),
    _g("gemm_k_below_64", 130, 24, 40, bn=64, bias=True, kernels=[fixed(64, 4)]),
    # >= one wave of output tiles: the persistent kernel
    _g("gemm_persistent", 4104, 2000, 520, bn=128, fams="EF", kernels=[persistent(128, 3)]),
    _g("gemm_persistent_nn_bias_relu_alpha2", 4104, 2000, 520, a_mn=True, b_mn=True, bn=128, bias=True, act=1,
       alpha=2.0, kernels=[persistent(128, 3)]),
    _g("gemm_persistent_bias_gelu", 4104, 2000, 520, bn=128, bias=True, act=2, outs=(BF16,),
       kernels=[persistent(128, 3)]),
    # cluster split-K with the DSMEM reduce; 576 = 9 k tiles: the host halves a cluster of 8 (and of 4) to 2
    _g("gemm_cluster2", 128, 512, 4608, bn=64, split_k=-2, kernels=[splitk(64)]),
    _g("gemm_cluster4", 128, 512, 4608, bn=64, split_k=-4, fams="EF", kernels=[splitk(64)]),
    _g("gemm_cluster8", 128, 512, 4608, bn=64, split_k=-8, fams="EF", kernels=[splitk(64)]),
    _g("gemm_cluster4_bn128_bias_relu", 200, 136, 1032, bn=128, split_k=-4, bias=True, act=1, kernels=[splitk(128)]),
    _g("gemm_cluster8_halved", 256, 256, 576, bn=64, split_k=-8, kernels=[splitk(64)]),
    # atomic split-K into a prefilled fp32 buffer (weight-gradient form); n_valid with a narrower output pitch (stem)
    _g("gemm_atomic_split7", 64, 576, 16384, a_mn=True, b_mn=True, split_k=7, accumulate=True, outs=(F32,),
       fams="EF", kernels=[fixed(64, 8)]),
    _g("gemm_n_valid_147_of_152", 64, 152, 4096, a_mn=True, b_mn=True, split_k=3, accumulate=True, n_valid=147,
       outs=(F32,), kernels=[fixed(64, 8)]),
    # the SIMT fallback: an operand pitch that is not a multiple of 8, and forced on aligned operands
    _g("gemm_simt_pitch10_bias", 256, 512, 10, bias=True, kernels=[SIMT]),
    _g("gemm_simt_forced_bias_gelu", 96, 72, 200, bias=True, act=2, simt=True, kernels=[SIMT]),
    _g("gemm_simt_forced_accumulate_alpha2", 96, 72, 200, a_mn=True, b_mn=True, simt=True, accumulate=True,
       alpha=2.0, alpha_f=0.3, outs=(F32,), fams="EF", kernels=[SIMT]),
    # epilogues
    _g("gemm_bias_relu_alpha_half", 300, 520, 328, bn=128, bias=True, act=1, alpha=0.5, kernels=[fixed(128, 6)]),
    _g("gemm_bias_gelu_bn64", 300, 200, 200, bn=64, bias=True, act=2, kernels=[fixed(64, 4)]),
    _g("gemm_alpha", 296, 136, 456, bn=128, alpha=2.0, alpha_f=0.3, fams="EF", kernels=[fixed(128, 6)]),
    _g("gemm_stats_fixed", 1000, 72, 128, bn=64, stats=True, outs=(BF16,), kernels=[fixed(64, 4)]),
    _g("gemm_stats_persistent", 4104, 2000, 520, bn=128, stats=True, outs=(BF16,), kernels=[persistent(128, 3)]),
    _g("gemm_stats_cluster4", 500, 200, 4608, bn=64, split_k=-4, stats=True, outs=(BF16,), kernels=[splitk(64)]),
    _g("gemm_affine_fixed_residual_relu", 300, 136, 328, bn=128, affine="residual_relu", outs=(BF16,),
       kernels=[fixed(128, 6, affine=1)]),
    _g("gemm_affine_cluster4", 128, 256, 2304, bn=64, split_k=-4, affine="plain", outs=(BF16,),
       kernels=[splitk(64, affine=1)]),
    # strided-batched GEMM as attention uses it: scores = Q K^T / 8 over (batch, head), then P V; >= 2 waves of tiles
    # take the persistent kernel, 3 x 5 problems the fixed one
    _b("batched_qk_persistent", "qk", 12, 24, 128, 64, kernels=[persistent(128, 3)]),
    _b("batched_pv_persistent", "pv", 12, 24, 128, 64, fams="EF", kernels=[persistent(64, 5)]),
    _b("batched_qk_odd", "qk", 3, 5, 96, 64, kernels=[fixed(128, 6)]),
    _b("batched_pv_odd", "pv", 3, 5, 96, 64, kernels=[fixed(64, 8)]),
    # every conv_plan form through F.conv_fwd
    _c("plan_centre", "plan", 126, 1, 1, 512, 256, 3, 1, 1, form="centre", kernels=[fixed(64, 8)]),
    _c("plan_pointwise", "plan", 6, 8, 8, 128, 256, 1, 1, 0, form="pointwise", kernels=[fixed(64, 4)]),
    _c("plan_implicit", "plan", 3, 4, 4, 256, 256, 3, 1, 1, form="implicit", fams="EF", kernels=[splitk(64, conv=1)]),
    _c("plan_im2col_stem", "plan", 6, 32, 32, 3, 64, 7, 2, 3, form="im2col", kernels=[fixed(64, 4)]),
    _c("plan_im2col_cin24", "plan", 3, 8, 8, 24, 64, 3, 1, 1, form="im2col", kernels=[fixed(64, 4)]),
    # im2col-mode implicit forward, cluster split-K 1 / 2 / 4 / 8, and a 1x1 stride-2 conv on the shallow ring
    _c("fwd_im2col_cluster1", "fwd", 6, 4, 4, 256, 128, 3, 1, 1, path="im2col", cluster_k=1, bn=64,
       kernels=[fixed(64, 8, conv=1)]),
    _c("fwd_im2col_cluster2", "fwd", 6, 4, 4, 256, 128, 3, 1, 1, path="im2col", cluster_k=2, bn=128,
       kernels=[splitk(128, conv=1)]),
    _c("fwd_im2col_cluster4_stats", "fwd", 6, 4, 4, 256, 128, 3, 1, 1, path="im2col", cluster_k=4, bn=64, stats=True,
       kernels=[splitk(64, conv=1)]),
    _c("fwd_im2col_cluster8", "fwd", 6, 4, 4, 256, 128, 3, 1, 1, path="im2col", cluster_k=8, bn=128, fams="EF",
       kernels=[splitk(128, conv=1)]),
    _c("fwd_1x1_s2_shallow", "fwd", 126, 8, 8, 128, 128, 1, 2, 0, cluster_k=1, bn=128,
       kernels=[fixed(128, 3, conv=1)]),
    # the halo kernel, stride 1 over 64 channels (8x8), cluster sizes 1 / 2 / 4, forward with statistics and input
    # gradient; then stride 1 over 128 channels (4x4) and stride 2 over 64 channels (8x8 -> 4x4)
    _c("halo_fwd_mc4_stats", "fwd", 128, 8, 8, 64, 64, 3, 1, 1, path="halo", mc=4, stats=True, fams="EF",
       kernels=[halo(0, 1, 1)]),
    _c("halo_fwd_mc2_stats", "fwd", 126, 8, 8, 64, 64, 3, 1, 1, path="halo", mc=2, stats=True, kernels=[halo(0, 1, 1)]),
    _c("halo_fwd_mc1_stats", "fwd", 3, 8, 8, 64, 64, 3, 1, 1, path="halo", mc=1, stats=True, kernels=[halo(0, 1, 1)]),
    _c("halo_dgrad_mc4", "dgrad", 128, 8, 8, 64, 64, 3, 1, 1, path="halo", mc=4, kernels=[halo(1, 1, 1)]),
    _c("halo_dgrad_mc2", "dgrad", 126, 8, 8, 64, 64, 3, 1, 1, path="halo", mc=2, fams="EF", kernels=[halo(1, 1, 1)]),
    _c("halo_dgrad_mc1", "dgrad", 1, 8, 8, 64, 64, 3, 1, 1, path="halo", mc=1, kernels=[halo(1, 1, 1)]),
    _c("wide_s1_fwd_mc8_stats", "fwd", 128, 4, 4, 128, 128, 3, 1, 1, path="halo", mc=8, stats=True, fams="EF",
       kernels=[halo(0, 2, 1)]),
    _c("wide_s1_fwd_mc2", "fwd", 126, 4, 4, 128, 128, 3, 1, 1, path="halo", mc=2, kernels=[halo(0, 2, 1)]),
    _c("wide_s1_fwd_mc1", "fwd", 1, 4, 4, 128, 128, 3, 1, 1, path="halo", mc=1, kernels=[halo(0, 2, 1)]),
    _c("wide_s2_fwd_mc4_stats", "fwd", 128, 8, 8, 64, 128, 3, 2, 1, path="halo", mc=4, stats=True,
       kernels=[halo(0, 1, 2)]),
    _c("wide_s2_fwd_mc1", "fwd", 3, 8, 8, 64, 128, 3, 2, 1, path="halo", mc=1, kernels=[halo(0, 1, 2)]),
    _c("wide_dgrad_mc4", "dgrad", 128, 4, 4, 128, 128, 3, 1, 1, path="halo", mc=4, fams="EF",
       kernels=[halo(1, 2, 1)]),
    _c("wide_dgrad_mc2", "dgrad", 6, 4, 4, 128, 128, 3, 1, 1, path="halo", mc=2, kernels=[halo(1, 2, 1)]),
    _c("wide_dgrad_mc1", "dgrad", 1, 4, 4, 128, 128, 3, 1, 1, path="halo", mc=1, kernels=[halo(1, 2, 1)]),
    # stride-1 implicit input gradient (im2col mode): cluster split-K 4 by default, and the single-pass kernel
    _c("dgrad_s1_im2col_cluster", "dgrad", 126, 2, 2, 256, 256, 3, 1, 1, path="im2col", kernels=[splitk(64, conv=3)]),
    _c("dgrad_s1_im2col_cluster1", "dgrad", 6, 8, 8, 64, 64, 3, 1, 1, path="im2col", cluster_k=1,
       kernels=[fixed(64, 8, conv=3)]),
    # stride-2 sub-pixel input gradient: odd maps, and k = 1 (classes without taps write zeros)
    _c("dgrad_s2_7x7", "dgrad", 3, 7, 7, 64, 128, 3, 2, 1, fams="EF", kernels=[fixed(64, 8, conv=4)]),
    _c("dgrad_s2_5x9", "dgrad", 3, 5, 9, 64, 128, 3, 2, 1, kernels=[fixed(64, 8, conv=4)]),
    _c("dgrad_s2_k1", "dgrad", 6, 8, 8, 64, 128, 1, 2, 0, kernels=[fixed(64, 8, conv=4)]),
    _c("dgrad_s2_8x8_n126", "dgrad", 126, 8, 8, 64, 128, 3, 2, 1, kernels=[fixed(64, 8, conv=4)]),
    # implicit weight gradient, accumulated into a prefilled buffer; batch 128 on 4x4 takes atomic split-K 3
    _c("wgrad_s1", "wgrad", 6, 8, 8, 64, 64, 3, 1, 1, kernels=[fixed(64, 8, conv=2)]),
    _c("wgrad_s2", "wgrad", 3, 8, 8, 64, 128, 3, 2, 1, kernels=[fixed(64, 8, conv=2)]),
    _c("wgrad_split3", "wgrad", 128, 4, 4, 128, 128, 3, 1, 1, fams="EF", kernels=[fixed(64, 8, conv=2)]),
    # eval-mode BatchNorm epilogue on the implicit forward (the halo kernel does not take it)
    _c("fwd_affine_cluster4", "fwd", 6, 4, 4, 128, 128, 3, 1, 1, affine="residual_relu",
       kernels=[splitk(64, conv=1, affine=1)]),
    _c("fwd_affine_single_pass", "fwd", 3, 8, 8, 64, 64, 3, 1, 1, affine="plain", cluster_k=1,
       kernels=[fixed(64, 8, conv=1, affine=1)]),
]
CASE_IDS = [c.id for c in CASES]
assert len(set(CASE_IDS)) == len(CASE_IDS)


# ------------------------------------------------------------------------------------------------ data
def _signs(shape, g):
    return torch.where(torch.rand(shape, generator=g) < 0.5, -1.0, 1.0).double()


def _ints(shape, density, g):
    """Entries in {-2, -1, 0, 1, 2}: nonzero with probability ``density``, then magnitude 1 or 2 and a random sign."""
    mag = torch.where(torch.rand(shape, generator=g) < 0.5, 1.0, 2.0).double()
    return mag * _signs(shape, g) * (torch.rand(shape, generator=g) < density).double()


def _hot_mag(shape, g):
    return torch.where(torch.rand(shape, generator=g) < 0.75, 2.0, 1.0).double()


def _density(k, stats_rows=0):
    """About 1200 expected per output of sum |a||b| (a term is 2.25 d^2 on average); with ``stats_rows`` also the
    column sums of squares of the output (6.25 d^2 K per row) under 2^22."""
    d = min(1.0, math.sqrt(1200.0 / (2.25 * k)))
    if stats_rows:
        d = min(d, math.sqrt(2 ** 22 / (6.25 * k * stats_rows)))
    return d


def _hot_rows(n, g):
    return torch.unique(torch.cat([torch.tensor([0, n - 1]), torch.randperm(n, generator=g)[:6]]))


def _plant_gemm(A, B, hot, g):
    """Hot rows of A and of B share one sign pattern over ``hot`` k indices and are zero elsewhere: their products are
    positive and the results of order 3 * hot (at most 4 * hot)."""
    K = A.shape[1]
    h = min(K, hot)
    ks = torch.randperm(K, generator=g)[:h]
    s = _signs(h, g)
    for T in (A, B):
        rows = _hot_rows(T.shape[0], g)
        T[rows] = 0.0
        T[rows[:, None], ks[None, :]] = s * _hot_mag((len(rows), h), g)


def _plant_conv(X, Wr, hot, g, imgs):
    """Convolution form of :func:`_plant_gemm`: images ``imgs`` of the gathered tensor ``X [n, h, w, c]`` and hot rows
    of ``Wr [rows, kh, kw, c]`` (``c`` = the reduction channel) share one sign per channel over ``hot / taps``
    channels and are zero on the others."""
    c, taps = X.shape[3], Wr.shape[1] * Wr.shape[2]
    hc = min(c, max(1, hot // taps))
    chans = torch.randperm(c, generator=g)[:hc]
    s = _signs(hc, g)
    for i in imgs:
        X[i] = 0.0
        X[i][:, :, chans] = s * _hot_mag(X.shape[1:3] + (hc,), g)
    for r in _hot_rows(Wr.shape[0], g).tolist():
        Wr[r] = 0.0
        Wr[r][:, :, chans] = s * _hot_mag(Wr.shape[1:3] + (hc,), g)


def _operand(shape, fam, density, g):
    return _ints(shape, density, g) if fam == "E" else torch.randn(shape, generator=g).to(BF16).double()


def _epilogue_data(c, fam, M, N, g):
    o, d = c.opts, {}
    if o.get("bias"):
        lim = 3 if o.get("act") == 2 else 300     # GELU: keep the pre-activations where GELU is not linear or zero
        d["bias"] = (torch.randint(-lim, lim + 1, (N,), generator=g).double() if fam == "E"
                     else torch.randn(N, generator=g).double())
    if o.get("accumulate"):
        d["prefill"] = (torch.randint(-64, 65, (M, N), generator=g).double() if fam == "E"
                        else torch.randn(M, N, generator=g).double())
    if o.get("stats"):
        d["stats_prefill"] = torch.randint(-64, 65, (2 * N,), generator=g).double()
    if o.get("affine"):
        d["scale"] = torch.pow(2.0, torch.randint(-2, 2, (N,), generator=g).double())
        d["shift"] = torch.randint(-64, 65, (N,), generator=g).double()
        if o["affine"] == "residual_relu":
            d["residual"] = torch.randint(-64, 65, (M, N), generator=g).double()
    return d


def _alpha(c, fam):
    a = c.opts.get("alpha_f", c.opts.get("alpha", 1.0)) if fam == "F" else c.opts.get("alpha", 1.0)
    return float(torch.tensor(a, dtype=F32))      # the kernel's fp32 alpha


@functools.lru_cache(maxsize=None)
def _data(cid, fam):
    """CPU float64 operands of one case (every value exact in bf16) and its epilogue inputs."""
    c = CASES[CASE_IDS.index(cid)]
    g = torch.Generator().manual_seed(CASE_IDS.index(cid) * 2 + (fam == "F"))
    geo, o = c.geo, c.opts
    if c.op == "gemm":
        M, N, K = geo["M"], geo["N"], geo["K"]
        dens = _density(K, M if o.get("stats") else 0)
        A, B = _operand((M, K), fam, dens, g), _operand((N, K), fam, dens, g)
        if fam == "E":
            _plant_gemm(A, B, 100 if o.get("stats") else 960, g)
        if o.get("n_valid"):
            B[o["n_valid"]:] = 0.0        # the zero K-padding rows of a stem weight gradient
        return dict(A=A, B=B, **_epilogue_data(c, fam, M, o.get("n_valid") or N, g))
    if c.op == "batched":
        Bt, H, S, dh = geo["B"], geo["H"], geo["S"], geo["dh"]
        D = H * dh
        qkv = _operand((Bt * S, 3 * D), fam, _density(S if geo["which"] == "pv" else dh), g)
        probs = _operand((Bt, H, S, S), fam, _density(S), g) if geo["which"] == "pv" else None
        if fam == "E" and probs is not None:      # hot (query, head-dim) pairs of every (batch, head)
            V = qkv.view(Bt, S, 3, H, dh)[:, :, 2]
            for b in range(Bt):
                for h in range(H):
                    A, Bv = probs[b, h].clone(), V[b, :, h].t().contiguous()
                    _plant_gemm(A, Bv, 960, g)
                    probs[b, h], V[b, :, h] = A, Bv.t()
        return dict(qkv=qkv, probs=probs)
    n, h, w, cin, cout, k, s, p = (geo[x] for x in ("n", "h", "w", "cin", "cout", "k", "stride", "pad"))
    ho, wo = F.conv_out_size(h, k, s, p), F.conv_out_size(w, k, s, p)
    if c.op == "wgrad":
        dens = _density(n * ho * wo)
        return dict(x=_operand((n, h, w, cin), fam, dens, g), dy=_operand((n, ho, wo, cout), fam, dens, g),
                    prefill=(torch.randint(-64, 65, (cout, k * k * cin), generator=g).double() if fam == "E"
                             else torch.randn(cout, k * k * cin, generator=g).double()))
    dgrad = c.op == "dgrad"
    cg, rows, m = (cout, cin, n * h * w) if dgrad else (cin, cout, n * ho * wo)
    dens = _density(k * k * cg, m if o.get("stats") else 0)
    X = _operand((n, ho, wo, cout) if dgrad else (n, h, w, cin), fam, dens, g)
    Wr = _operand((rows, k, k, cg), fam, dens, g)          # one row per GEMM column, reduction channel last
    if fam == "E":
        _plant_conv(X, Wr, 100 if o.get("stats") else 960, g, [n - 1] if o.get("stats") or n == 1 else [0, n - 1])
    wt = (Wr.permute(3, 1, 2, 0) if dgrad else Wr).contiguous()          # [cout, kh, kw, cin]
    d = dict(w=wt)
    d["dy" if dgrad else "x"] = X
    d.update(_epilogue_data(c, fam, m, cin if dgrad else cout, g))
    return d


# ------------------------------------------------------------------------------------------------ float64 reference
def _nchw(t):
    return t.permute(0, 3, 1, 2)


def _oihw(w):
    return w.permute(0, 3, 1, 2)


def _gelu64(v):
    return 0.5 * v * (1.0 + torch.tanh(math.sqrt(2.0 / math.pi) * (v + 0.044715 * v ** 3)))


def _accumulator(c, d, absolute=False):
    """The case's GEMM result (``[rows, cols]`` float64) before any epilogue, or with ``absolute`` the same operation
    on |operands| (``sum_k |a_k b_k|``): an explicit matmul, batched matmul or torch float64 convolution."""
    ab = (lambda t: t.abs()) if absolute else (lambda t: t)
    geo = c.geo
    if c.op == "gemm":
        return (ab(d["A"]) @ ab(d["B"]).t())[:, : c.opts.get("n_valid") or geo["N"]]
    if c.op == "batched":
        Bt, H, S, dh = geo["B"], geo["H"], geo["S"], geo["dh"]
        qkv = ab(d["qkv"]).view(Bt, S, 3, H, dh).permute(2, 0, 3, 1, 4)          # [3, B, H, S, dh]
        if geo["which"] == "qk":
            return (qkv[0] @ qkv[1].transpose(-1, -2)).reshape(-1, S)              # [B H S, S]
        return (ab(d["probs"]) @ qkv[2]).permute(0, 2, 1, 3).reshape(Bt * S, H * dh)   # [B S, H dh]
    s, p, k = geo["stride"], geo["pad"], geo["k"]
    if c.op == "wgrad":
        shape = (geo["cout"], geo["cin"], k, k)
        dw = torch.nn.grad.conv2d_weight(_nchw(ab(d["x"])), shape, _nchw(ab(d["dy"])), s, p)
        return dw.permute(0, 2, 3, 1).reshape(geo["cout"], -1)
    w4 = _oihw(ab(d["w"]))
    if c.op == "dgrad":
        shape = (geo["n"], geo["cin"], geo["h"], geo["w"])
        dx = torch.nn.grad.conv2d_input(shape, w4, _nchw(ab(d["dy"])), s, p)
        return dx.permute(0, 2, 3, 1).reshape(-1, geo["cin"])
    return TF.conv2d(_nchw(ab(d["x"])), w4, None, s, p).permute(0, 2, 3, 1).reshape(-1, geo["cout"])


def _reference(c, d, fam):
    """``(out, pre)``: the float64 output of the case and the pre-activation GELU is applied to."""
    o = c.opts
    v = _accumulator(c, d) * _alpha(c, fam)
    if "bias" in d:
        v = v + d["bias"]
    pre = v
    if o.get("act") == 1:
        v = v.clamp_min(0.0)
    elif o.get("act") == 2:
        v = _gelu64(v)
    if o.get("affine"):
        v = v * d["scale"] + d["shift"] + d.get("residual", 0.0)
        if o["affine"] == "residual_relu":
            v = v.clamp_min(0.0)
    if "prefill" in d:
        v = d["prefill"] + v
    return v, pre


def _frexp_grid(r):
    """``|r| = q * ulp`` on the bf16 grid (8 significant bits, subnormal spacing below 2^-126)."""
    a = r.abs()
    _, e = torch.frexp(a)
    ulp = torch.ldexp(torch.ones_like(a), (e - 1).clamp_min(-126) - 7)       # exact, unlike pow on the GPU
    return a / ulp, ulp


def _round_bf16(r, mode="rne"):
    """float64 ``r`` rounded to bf16 (finite range): nearest-even, or the conversions a kernel must not use."""
    q, ulp = _frexp_grid(r)
    m = {"rne": torch.round, "trunc": torch.floor, "away": lambda t: torch.floor(t + 0.5),
         "up": torch.ceil}[mode](q)
    return torch.sign(r) * m * ulp


def _neighbour(r, rn):
    """The bf16 value next to ``rn = round(r)`` on ``r``'s side (``rn`` itself where ``r`` is exact)."""
    up = _round_bf16(r, "up")
    down = _round_bf16(r, "trunc")
    return torch.where(r.abs() > rn.abs(), up, torch.where(r.abs() < rn.abs(), down, rn))


# ------------------------------------------------------------------------------------------------ checks
def _mismatch(tag, got, ref, bad):
    idx = bad.nonzero()[:5].tolist()
    return "{}: {} of {} elements differ, first at {}: got {} want {}".format(
        tag, int(bad.sum()), bad.numel(), idx, [float(got[tuple(i)]) for i in idx], [float(ref[tuple(i)]) for i in idx])


def _check_exact(tag, got, ref):
    """fp32: equal to the float64 reference; bf16: equal to its round-to-nearest-even."""
    want = ref if got.dtype == F32 else _round_bf16(ref)
    g = got.double()
    bad = ~(g == want)
    assert not bad.any(), _mismatch(tag, g, want, bad)


def _check_window(tag, got, ref, window):
    """A bf16 ``got`` must be the correct rounding of some value within ``window`` of ``ref``: ``ref`` rounded to
    nearest-even where no bf16 midpoint lies that close, either neighbour of ``ref`` where one does, and more than one
    ulp away only where the window is wider than the bf16 spacing.  Returns the fraction of elements with a midpoint
    inside the window."""
    rn = _round_bf16(ref)
    nb = _neighbour(ref, rn)
    g = got.double()
    bad = ~((g >= _round_bf16(ref - window)) & (g <= _round_bf16(ref + window)))
    assert not bad.any(), _mismatch(tag, g, rn, bad)
    return float((((ref - 0.5 * (rn + nb)).abs() <= window) & (nb != rn)).double().mean())


def _check_gelu(tag, got, ref, pre):
    """Within ``2^-19 |pre|`` of the float64 GELU (bf16: the correct rounding of a value that close)."""
    window = 2.0 ** -19 * pre.abs()
    if got.dtype == F32:
        bad = ~((got.double() - ref).abs() <= window)
        assert not bad.any(), _mismatch(tag, got.double(), ref, bad)
    else:
        _check_window(tag, got, ref, window)


def _check_full_mantissa(tag, got, ref, absum):
    if got.dtype == F32:
        ratio = float((got.double() - ref).pow(2).mean().sqrt() / ref.pow(2).mean().sqrt())
        print("{}: rms ratio 2^{:.2f}".format(tag, math.log2(ratio) if ratio > 0 else -math.inf))
        assert ratio <= 2.0 ** -14, ratio
    else:
        frac = _check_window(tag, got, ref, 2.0 ** -18 * absum)
        g = got.double()
        off = g != _round_bf16(ref)
        # the least error before the bf16 rounding that explains each such element: its distance from the values
        # that round to `got`
        implied = ((g - ref).abs() - 0.5 * _frexp_grid(g)[1]).clamp_min(0.0) / absum
        worst = float(implied[off].max()) if off.any() else 0.0
        print("{}: {:.4%} of the elements within the window of a midpoint, {} not correctly rounded, worst implied "
              "error / sum|ab| = 2^{:.2f}".format(tag, frac, int(off.sum()), math.log2(worst) if worst > 0 else -math.inf))


def _group_nonzero(contrib, size):
    """``contrib [..., K]`` summed over consecutive groups of ``size`` along the last dim."""
    k = contrib.shape[-1]
    pad = (-k) % size
    return TF.pad(contrib, (0, pad)).reshape(contrib.shape[:-1] + ((k + pad) // size, size)).sum(-1)


def _sensitivity(c, d, g):
    """Random projections of each k group's contribution (GEMM: 16-wide k groups; convolutions: (tap, 16-channel
    group), where the tap can reach an output at all; weight gradients: 16-pixel groups): all must be nonzero."""
    geo = c.geo
    if c.op in ("gemm", "batched"):
        pairs = [(d["A"], d["B"])] if c.op == "gemm" else []
        if c.op == "batched":
            Bt, H, S, dh = geo["B"], geo["H"], geo["S"], geo["dh"]
            qkv = d["qkv"].view(Bt, S, 3, H, dh).permute(2, 0, 3, 1, 4)
            for b in range(Bt):
                for h in range(H):
                    pairs.append((qkv[0, b, h], qkv[1, b, h]) if geo["which"] == "qk"
                                 else (d["probs"][b, h], qkv[2, b, h].t()))
        out = []
        for A, B in pairs:
            u = torch.randn(A.shape[0], generator=g, dtype=F64)
            v = torch.randn(B.shape[0], generator=g, dtype=F64)
            out.append(_group_nonzero((u @ A) * (v @ B), 16))
        return torch.cat(out), None
    s, p = geo["stride"], geo["pad"]
    if c.op == "wgrad":
        x4, dy4 = _nchw(d["x"]), _nchw(d["dy"])
        V = torch.randn((geo["cout"], geo["cin"], geo["k"], geo["k"]), generator=g, dtype=F64)
        z = (TF.conv2d(x4, V, None, s, p) * dy4).sum(1)              # per output pixel, NHW order
        return _group_nonzero(z.reshape(-1), 16), None
    w4 = _oihw(d["w"])
    if c.op == "dgrad":
        U = torch.randn((geo["n"], geo["cin"], geo["h"], geo["w"]), generator=g, dtype=F64)
        G = torch.nn.grad.conv2d_weight(U, w4.shape, _nchw(d["dy"]), s, p)
        reach = torch.nn.grad.conv2d_weight(torch.ones_like(U), w4.shape, torch.ones_like(_nchw(d["dy"])), s, p)
        red = (1, 0)                                      # reduce over cin, group cout
    else:
        x4 = _nchw(d["x"])
        ho, wo = F.conv_out_size(geo["h"], geo["k"], s, p), F.conv_out_size(geo["w"], geo["k"], s, p)
        U = torch.randn((geo["n"], geo["cout"], ho, wo), generator=g, dtype=F64)
        G = torch.nn.grad.conv2d_weight(x4, w4.shape, U, s, p)
        reach = torch.nn.grad.conv2d_weight(torch.ones_like(x4), w4.shape, torch.ones_like(U), s, p)
        red = (0, 1)                                      # reduce over cout, group cin
    contrib = (G * w4).sum(red[0])                        # [channel, kh, kw]
    reach = reach.sum(red[0]) > 0
    return _group_nonzero(contrib.permute(1, 2, 0), 16), _group_nonzero(reach.permute(1, 2, 0).double(), 16) > 0


# ------------------------------------------------------------------------------------------------ CPU: the generator
def _bf16_outputs(c):
    if c.op in ("gemm", "batched"):
        return BF16 in c.opts["outs"]
    return c.op in ("plan", "fwd", "dgrad")


def _needs_big(c):
    """Bf16 cases whose operation can reach 256: attention scores (K = 64 head dims, alpha 1/8) stay below 32."""
    return _bf16_outputs(c) and not (c.op == "batched" and c.geo["which"] == "qk")


def test_generator_bounds_and_sensitivity():
    """Family E data of every case, in float64 on the CPU: the 2^12 bound, the 2^24 statistics bound, results above
    256 with ties that a truncating or ties-away bf16 conversion gets wrong, and every k group / tap contributing."""
    for c in CASES:
        d = _data(c.id, "E")
        for t in d.values():
            if t is not None:
                assert torch.equal(t, t.round()) or t is d.get("scale"), c.id
        bound = float(_accumulator(c, d, absolute=True).max())
        assert bound <= EXACT_BOUND, (c.id, bound)
        ref, _ = _reference(c, d, "E")
        if _needs_big(c):
            rne = _round_bf16(ref)
            assert (ref.abs() > 256).any(), (c.id, float(ref.abs().max()))
            assert (_round_bf16(ref, "trunc") != rne).any(), c.id
            assert (_round_bf16(ref, "away") != rne).any(), c.id
        if c.opts.get("stats"):
            y = _round_bf16(ref)
            sq = float((y * y).sum(0).max()) + 64
            assert sq < STATS_BOUND, (c.id, sq)
        groups, reach = _sensitivity(c, d, torch.Generator().manual_seed(7))
        if reach is not None:
            assert reach.any(), c.id
            groups = groups[reach]
        assert groups.numel() and bool((groups != 0).all()), (c.id, int((groups == 0).sum()), groups.numel())


def test_exact_checks_reject_dropped_terms_and_wrong_rounding():
    """The exact comparison fails against a reference with one k group or one tap dropped, and against bf16 outputs
    rounded by truncation or ties-away."""
    c = CASES[CASE_IDS.index("gemm_kk_bn128_deep")]
    d = _data(c.id, "E")
    ref, _ = _reference(c, d, "E")
    for g0 in (0, 7, 20):                                   # 16-wide k groups, the last one ragged (328 = 20.5 x 16)
        A = d["A"].clone()
        A[:, 16 * g0: 16 * g0 + 16] = 0.0
        dropped = A @ d["B"].t()
        for dt in (F32, BF16):
            got = dropped.to(dt)
            with pytest.raises(AssertionError):
                _check_exact("dropped k group", got, ref)
    for mode in ("trunc", "away"):
        got = _round_bf16(ref, mode).to(BF16)
        with pytest.raises(AssertionError):
            _check_exact(mode, got, ref)
    _check_exact("nearest-even", _round_bf16(ref).to(BF16), ref)
    for cid in ("halo_fwd_mc4_stats", "dgrad_s2_5x9"):
        c = CASES[CASE_IDS.index(cid)]
        d = dict(_data(cid, "E"))
        ref, _ = _reference(c, d, "E")
        for tap in (0, 4, 8):                                # one tap of the 3x3 filter dropped
            w = d["w"].clone()
            w[:, tap // 3, tap % 3, :] = 0.0
            got, _ = _reference(c, dict(d, w=w), "E")
            with pytest.raises(AssertionError):
                _check_exact("dropped tap", got.to(BF16), ref)


# ------------------------------------------------------------------------------------------------ GPU
def _guarded(rows, cols, dtype, dev, *, ldd=None, extra_rows=0, tail=67, prefill=None):
    """``[rows, cols]`` view (row pitch ``ldd``) of a buffer with ``extra_rows`` more rows and a tail, every element
    holding the NaN sentinel; returns ``(view, check)``: ``check()`` asserts the guard elements kept their bits."""
    ldd = ldd or cols
    idt, bits = SENTINEL[dtype]
    total = (rows + extra_rows) * ldd + tail
    buf = torch.full((total,), bits, dtype=idt, device=dev)
    view = buf[: rows * ldd].view(rows, ldd)[:, :cols].view(dtype)
    if prefill is not None:
        view.copy_(prefill)
    guard = torch.ones(total, dtype=torch.bool, device=dev)
    guard[: rows * ldd].view(rows, ldd)[:, :cols] = False

    def check(tag):
        changed = int((buf[guard] != bits).sum())
        assert changed == 0, "{}: {} guard elements overwritten".format(tag, changed)
    return view, check


def _affine_arg(d, dev, rows, cols):
    a = {"scale": d["scale"].to(dev, F32), "shift": d["shift"].to(dev, F32), "relu": "residual" in d}
    if "residual" in d:
        a["residual"] = d["residual"].to(dev, BF16).view(rows, cols)
    return a


def _run(c, d, fam, out_dtype, dev):
    """Launch the case; returns ``({name: output}, [guard checks])``."""
    geo, o = c.geo, c.opts
    bf = lambda t: t.to(dev, BF16).contiguous()          # noqa: E731  (exact: every operand is a bf16 value)
    outs, checks = {}, []
    if c.op == "gemm":
        M, K = geo["M"], geo["K"]
        N = o.get("n_valid") or geo["N"]
        ldd = o.get("n_valid") or (F.round_up(N, 8) + 8)
        out, chk = _guarded(M, N, out_dtype, dev, ldd=ldd, extra_rows=5, prefill=d.get("prefill"))
        checks.append(chk)
        kw = dict(a_mn=geo["a_mn"], b_mn=geo["b_mn"], out=out, split_k=geo["split_k"], force_bn=geo["bn"],
                  alpha=_alpha(c, fam), act=o.get("act", 0), accumulate=bool(o.get("accumulate")),
                  force_simt=bool(o.get("simt")), n_valid=o.get("n_valid"))
        if "bias" in d:
            kw["bias"] = d["bias"].to(dev, F32)
        if o.get("stats"):
            kw["col_stats"], chk = _guarded(1, 2 * N, F32, dev, prefill=d["stats_prefill"].view(1, -1))
            kw["col_stats"] = kw["col_stats"].view(-1)
            checks.append(chk)
        if o.get("affine"):
            kw["affine"] = _affine_arg(d, dev, M, N)
        a = bf(d["A"].t() if geo["a_mn"] else d["A"])
        b = bf(d["B"].t() if geo["b_mn"] else d["B"])
        assert F.gemm(a, b, **kw) is out
        outs["y"] = out
        if o.get("stats"):
            outs["stats"] = kw["col_stats"]
        return outs, checks
    if c.op == "batched":
        Bt, H, S, dh = geo["B"], geo["H"], geo["S"], geo["dh"]
        D = H * dh
        qkv = bf(d["qkv"])
        if geo["which"] == "qk":
            out, chk = _guarded(Bt * H * S, S, out_dtype, dev)
            F.gemm_batched(qkv, qkv[:, D:], out, M=S, N=S, K=dh, lda=3 * D, ldb=3 * D, ldd=S, a_mn=False, b_mn=False,
                           n_outer=Bt, n_inner=H, a_strides=(S * 3 * D, dh), b_strides=(S * 3 * D, dh),
                           d_strides=(H * S * S, S * S), alpha=_alpha(c, fam))
        else:
            out, chk = _guarded(Bt * S, D, out_dtype, dev)
            F.gemm_batched(bf(d["probs"]), qkv[:, 2 * D:], out, M=S, N=dh, K=S, lda=S, ldb=3 * D, ldd=D, a_mn=False,
                           b_mn=True, n_outer=Bt, n_inner=H, a_strides=(H * S * S, S * S),
                           b_strides=(S * 3 * D, dh), d_strides=(S * D, dh))
        outs["y"], checks = out, [chk]
        return outs, checks
    n, h, w, cin, cout, k, s, p = (geo[x] for x in ("n", "h", "w", "cin", "cout", "k", "stride", "pad"))
    ho, wo = F.conv_out_size(h, k, s, p), F.conv_out_size(w, k, s, p)
    if c.op == "wgrad":
        dw, chk = _guarded(cout, k * k * cin, F32, dev, prefill=d["prefill"])
        assert F.conv_igemm_wgrad_(bf(d["dy"]).view(-1, cout), bf(d["x"]), dw, k, k, s, p)
        return {"y": dw}, [chk]
    w2d = bf(d["w"].reshape(cout, -1))
    if c.op == "dgrad":
        dx, chk = _guarded(n * h * w, cin, BF16, dev)
        r = F.conv_igemm_dgrad(bf(d["dy"]), w2d, (n, h, w, cin), k, k, p, stride=s, out=dx.view(n, h, w, cin),
                               path=o.get("path"), mc=o.get("mc"), cluster_k=o.get("cluster_k"))
        assert r is not None and r.data_ptr() == dx.data_ptr()
        return {"y": dx}, [chk]
    if c.op == "plan":
        plan = F.conv_plan(n, h, w, cin, cout, k, k, s, p)
        assert plan.form == o["form"]
        if plan.form == "im2col":          # the weights carry the GEMM's zero K padding (F.im2col_k)
            w2d = TF.pad(w2d, (0, plan.K - w2d.shape[1]))
        y, _ = F.conv_fwd(bf(d["x"]), w2d, plan)
        return {"y": y}, []
    M = n * ho * wo
    y, chk = _guarded(M, cout, BF16, dev)
    checks.append(chk)
    kw = dict(out=y, path=o.get("path"), mc=o.get("mc"), cluster_k=o.get("cluster_k"), force_bn=o.get("bn", 0))
    if o.get("stats"):
        st, chk = _guarded(1, 2 * cout, F32, dev, prefill=d["stats_prefill"].view(1, -1))
        kw["col_stats"] = st.view(-1)
        checks.append(chk)
    if o.get("affine"):
        kw["affine"] = _affine_arg(d, dev, M, cout)
    assert F.conv_igemm_fwd(bf(d["x"]), w2d, k, k, s, p, **kw) is y
    outs["y"] = y
    if o.get("stats"):
        outs["stats"] = kw["col_stats"]
    return outs, checks


def _out_dtypes(c):
    if c.op in ("gemm", "batched"):
        return c.opts["outs"]
    return (F32,) if c.op == "wgrad" else (BF16,)


@pytest.fixture(scope="module")
def dev():
    F.load()
    return torch.device("cuda:0")


def _on(d, dev):
    return {k: (v.to(dev) if v is not None else None) for k, v in d.items()}


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=CASE_IDS)
def test_exact_integer_operands(case, dev):
    d = _data(case.id, "E")
    ref, pre = _reference(case, _on(d, dev), "E")
    for dt in _out_dtypes(case):
        outs, checks = _run(case, d, "E", dt, dev)
        torch.cuda.synchronize()
        tag = "{} {}".format(case.id, dt)
        got = outs["y"].reshape(ref.shape)
        if case.opts.get("act") == 2:
            _check_gelu(tag, got, ref, pre)
        else:
            _check_exact(tag, got, ref)
        if "stats" in outs:
            y = _round_bf16(ref)
            want = torch.cat([y.sum(0), (y * y).sum(0)]) + d["stats_prefill"].to(dev)
            _check_exact(tag + " column statistics", outs["stats"], want)
        for chk in checks:
            chk(tag)


@pytest.mark.gpu
@pytest.mark.parametrize("case", [c for c in CASES if "F" in c.fams], ids=[c.id for c in CASES if "F" in c.fams])
def test_full_mantissa_operands(case, dev):
    d = _data(case.id, "F")
    dd = _on(d, dev)
    ref, _ = _reference(case, dd, "F")
    absum = _accumulator(case, dd, absolute=True) * abs(_alpha(case, "F"))
    if "prefill" in dd:
        absum = absum + dd["prefill"].abs()
    for dt in _out_dtypes(case):
        outs, checks = _run(case, d, "F", dt, dev)
        torch.cuda.synchronize()
        tag = "{} {} (F)".format(case.id, dt)
        _check_full_mantissa(tag, outs["y"].reshape(ref.shape), ref, absum)
        for chk in checks:
            chk(tag)


_KERNEL = re.compile(r"(gemm_bf16_fixed_kernel|gemm_bf16_persistent_kernel|gemm_bf16_splitk_kernel|gemm_simt_kernel|"
                     r"conv_halo_kernel)(?:<([^>]*)>)?")


def _kernel_key(name):
    m = _KERNEL.search(name)
    if m is None:
        return None
    args = [{"true": "1", "false": "0"}.get(a, a) for a in
            (re.sub(r"^\(\w+\)", "", x.strip()) for x in (m.group(2) or "").split(","))]
    base = m.group(1)
    if base == "gemm_simt_kernel":
        return SIMT
    if base == "gemm_bf16_fixed_kernel":
        return fixed(*(int(args[i]) for i in (0, 1, 2, 4)))
    if base == "gemm_bf16_splitk_kernel":
        return splitk(int(args[0]), int(args[2]), int(args[3]), int(args[1]))
    if base == "gemm_bf16_persistent_kernel":
        return persistent(int(args[0]), int(args[1]))
    return halo(int(args[0]), int(args[1]), int(args[2]))


def test_kernel_key_parses_demangled_names():
    assert _kernel_key("void b200::gemm_bf16_fixed_kernel<128, 6, 1, false, true, false, false, false>"
                       "(CUtensorMap_st, CUtensorMap_st, b200::GemmParams)") == fixed(128, 6, 1, 1)
    assert _kernel_key("void b200::gemm_bf16_splitk_kernel<64, true, 3, false>(CUtensorMap_st, CUtensorMap_st, "
                       "b200::GemmParams)") == splitk(64, 3, 0)
    assert _kernel_key("void b200::conv_halo_kernel<(bool)1, 2, 1>(CUtensorMap_st, CUtensorMap_st, "
                       "b200::HaloParams)") == halo(1, 2, 1)
    assert _kernel_key("b200::gemm_simt_kernel(__nv_bfloat16 const*, ...)") == SIMT
    assert _kernel_key("void b200::conv_halo_kernel<false, 1, 1>(CUtensorMap_st, CUtensorMap_st, b200::HaloParams)") \
        == halo(0, 1, 1)


@pytest.mark.gpu
def test_case_table_reaches_every_kernel_instantiation(dev):
    """Each case's first output type under torch.profiler: every kernel instantiation the table names must appear, so
    a dispatch change that moves cases onto another kernel fails here instead of leaving a branch untested.
    (``force_bn=256`` runs as 128: the host clamps BN, and no 256-wide instantiation exists.)"""
    from torch.profiler import ProfilerActivity, profile
    want = set().union(*(c.kernels for c in CASES))
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for c in CASES:
            _run(c, _data(c.id, "E"), "E", _out_dtypes(c)[0], dev)
        torch.cuda.synchronize()
    seen = {_kernel_key(e.name) for e in prof.events()} - {None}
    assert want <= seen, sorted(want - seen)
    assert {"fixed<64,4,0,0>", "fixed<64,8,0,0>", "fixed<128,3,0,0>", "fixed<128,6,0,0>", "persistent<128,3>",
            "persistent<64,5>", "splitk<64,1,0,0>", "splitk<128,1,0,0>", SIMT, halo(0, 1, 1),
            halo(1, 1, 1)} <= want
