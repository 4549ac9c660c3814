"""The BatchNorm, LayerNorm and softmax kernels (csrc/norm.cu) against float64, at their dispatch branches and edges.
Every case is built on the CPU from a seeded generator and calls one entry point of the extension directly.  The
float64 reference follows each kernel's documented formula; it never calls a kernel or PyTorch's bf16 path.

Family E (exact).  Activations, gradients and residuals are small integers; gamma, beta, running statistics and the
prefilled accumulators are dyadic (k 2^-j with k of at most two bits); the backward kernels' ``mean`` is an integer
and ``rstd`` a power of two.  Where the forward statistics are computed, the row count (BatchNorm) or C (LayerNorm) is
a power of two and the generator moves single elements by one so that every column (row) mean is a multiple of 1/4.
The generator asserts that every sum these produce is a dyadic below 2^24 (``EXACT_BOUND``).  So, in any summation
order (atomics, DSMEM, shuffles):
* the fp32 sums, ``save_mean``, LayerNorm ``mean``, dgamma / dbeta and the accumulation into prefilled buffers equal
  float64 exactly;
* dx, dres, dz and the softmax gradient equal the float64 value rounded to nearest-even.  The generator asserts that
  some of these fall on bf16 rounding ties, so a ties-away conversion fails too;
* ``save_rstd`` / ``rstd`` are within 2 fp32 ulp (the documented ``rsqrtf`` error) of ``1/sqrt(fp32(var + eps))``.
The rstd that the kernel saved is then used to compute the float64 reference of y, so that rsqrt's error cannot hide anything else.
y itself is not exact: ``gamma * rstd``, ``mean * gamma * rstd``, the fma and the residual add round in fp32.  y must
be the correct bf16 rounding of a value within ``w = 8u (|x s| + |mean s| + |beta| + |res|)`` of the reference
(``u = 2^-24``, ``s = gamma rstd``; four fp32 roundings, twice over).  The stem pair is exact bit for bit: its cases
have zero column means and gamma = +-2^j, so the fp32 candidate ``fma(z, s, beta)`` is emulated exactly, then rounded
to fp32 and to bf16 as the kernel does.  The reference takes the first tap in raster order that has the strictly
largest bf16 value, and ``argmax`` must equal it.  Where a divisor is not a power of two (ragged row counts, C = 100
or 768, stem maps with odd H and W), the quotient rounds.  The outputs that depend on it then get the elementwise
window ``8u`` times the magnitudes they are built from, and rstd one more ulp.

Family F (full mantissa).  Operands are ``randn`` rounded to bf16.  The longest chain of dependent fp32 additions in
any reduction here is below 2^10 (rows per thread + partials per CTA + one atomic per CTA), so a correct fp32 sum is
within ``2^-14 sum|t|``.  A bf16 rounding of any partial (2^-9) or a lost term fails this bound.  Per kernel:
* sums, dgamma, dbeta: ``|got - ref| <= 2^-14 sum|t|``;
* save_mean / LayerNorm mean, from the kernel's own sums: ``4u |mean|`` (reciprocal and product; plus ``2^-14
  sum|x| / C`` for LayerNorm, whose sum is internal);
* rstd: 2 ulp plus ``1/2 |dvar| / (var + eps)`` relative, with ``|dvar| <= 6u (E[x^2] + mean^2)`` (BatchNorm, from the
  kernel's sums) or ``2^-14 E[(x - mean)^2]`` (LayerNorm);
* y (BatchNorm, LayerNorm), with the kernel's mean and rstd: the window ``w`` above;
* dx, dz: ``|gamma rstd| (8u (|g| + |mean_g| + |xhat mean_gx|) + e_g / n + |xhat| e_gx / n)``, where e is the 2^-14
  bound of the two internal sums and n the row count (C for LayerNorm);
* softmax: ``p_i u (16 + C + 2 a_i + sum_j p_j (8 + 2 a_j))`` relative to p, ``a_j = |x_j scale| + |x_j scale - max|``:
  the exponent's argument rounds twice, ``__expf`` is within 2^-21, the row sum has at most C terms.  Softmax backward
  is exact in family E; in F it gets ``8u`` of its terms plus the 2^-14 bound of its row sum.
Each F case prints, per output, the worst error as a fraction of its window (``pytest -rP``; a bf16 output counts only
where it is not the nearest-even rounding of the reference).  Measured on one H100 80GB HBM3 at a 700 W power limit:
* sums 0.016, save_mean 0.32, save_rstd 0.26, y 0.10, running statistics 0.23 (BatchNorm and stem);
* dgamma / dbeta 0.0018, dx / dz 0.0054 (BatchNorm, stem, LayerNorm);
* LayerNorm mean 0.0006, rstd 0.0055, y 0.022; softmax p 0 (every element correctly rounded), dx 0.0011.
With |mean| = 16, 63 and 230 std, the statistics lose precision to ``E[x^2] - mean^2``: the measured rstd relative
error is 2^-14.1, 2^-9.9 and 2^-5.8 against the data's float64 statistics (bounds 2^-6.9, 2^-2.9 and 2^0.8 from the
2^-14 chain and 6u of ``E[x^2] / var``).

Every output is written into a view of a larger buffer prefilled with a NaN bit pattern (a head where the case
misaligns its tensors, and a tail): the guard elements must keep their bits, and an element the kernel never writes
stays NaN and fails the comparison."""
import json
import math
import os
import re
import tempfile
from collections import namedtuple

import pytest
import torch

BF16, F32, F64 = torch.bfloat16, torch.float32, torch.float64
U = 2.0 ** -24                   # fp32 unit roundoff
CHAIN = 2.0 ** -14               # a correct fp32 reduction here is within CHAIN * sum|t|
EXACT_BOUND = 2 ** 24            # every family-E sum is a dyadic whose numerator stays below this
SENTINEL = {BF16: (torch.int16, 0x7FC1), F32: (torch.int32, 0x7FC00BAD), torch.uint8: (torch.uint8, 0xFE),
            torch.int64: (torch.int64, 0x7FF0DEAD)}
EPS, MOM = 1e-5, 0.25

Case = namedtuple("Case", "id op geo fams kernels")


# ------------------------------------------------------------------------------------------------ the case table
def _bnf(cid, rows, C, *, fams="E", kernels=(), **o):
    """bn_stats into a prefilled buffer, then bn_apply (training unless ``train=False``)."""
    geo = dict(rows=rows, C=C, train=True, res=False, relu=False, affine=True, offset=0, const=False, shift=0.0)
    geo.update(o)
    return Case(cid, "bn_fwd", geo, fams, frozenset(kernels))


def _bnb(cid, rows, C, *, fams="E", kernels=(), **o):
    """BatchNorm backward: ``mc`` set -> bn_bwd_cluster with that max_cluster, else bn_bwd_reduce + bn_bwd_apply."""
    geo = dict(rows=rows, C=C, mc=None, relu=True, dy_b=False, dres=True, affine=True, offset=0)
    geo.update(o)
    return Case(cid, "bn_bwd", geo, fams, frozenset(kernels))


def _stem(cid, N, H, W, C, *, fams="E", kernels=("bn_relu_maxpool", "bn_maxpool_bwd_reduce", "bn_maxpool_bwd_apply"),
          **o):
    geo = dict(N=N, H=H, W=W, C=C, k=3, s=2, p=1, dy_b=False, dead=False)
    geo.update(o)
    return Case(cid, "stem", geo, fams, frozenset(kernels))


def _row(cid, op, rows, C, *, fams="E", kernels=(), **o):
    geo = dict(rows=rows, C=C, offset=0, res=False, scale=1.0, mask=False, const=False)
    geo.update(o)
    return Case(cid, op, geo, fams, frozenset(kernels))


def clu(it, s):
    return "bn_bwd_cluster<{}>/S{}".format(it, s)


def vec(name, lpr, vpl):
    return "{}_vec<{},{}>".format(name, lpr, vpl)


def _ln(cid, rows, C, lv=None, **o):
    k = [vec("layernorm_fwd", *lv), vec("layernorm_bwd", *lv)] if lv else ["layernorm_fwd", "layernorm_bwd"]
    return _row(cid, "ln", rows, C, kernels=k, **o)


def _sm(cid, rows, C, lv=None, **o):
    k = [vec("softmax_fwd", *lv), vec("softmax_bwd", *lv)] if lv else ["softmax_fwd", "softmax_bwd"]
    return _row(cid, "sm", rows, C, kernels=k, **o)


VS, SS, AP = "bn_stats_vec", "bn_stats", "bn_apply"
CASES = [
    # statistics + apply: vectorised column reduction at C/8 = 1, 2, 8, 256; scalar at C = 24, 40 and when misaligned
    _bnf("bn_c64_res_relu", 8192, 64, res=True, relu=True, fams="EF", kernels=[VS, AP]),
    _bnf("bn_c8", 4096, 8, kernels=[VS, AP]),
    _bnf("bn_c16_relu", 4096, 16, relu=True, kernels=[VS, AP]),
    _bnf("bn_c2048", 1024, 2048, fams="EF", kernels=[VS, AP]),
    _bnf("bn_c24_scalar", 1024, 24, fams="EF", kernels=[SS, AP]),
    _bnf("bn_c40_scalar_ragged", 999, 40, kernels=[SS, AP]),
    _bnf("bn_c64_misaligned", 2048, 64, offset=2, kernels=[SS, AP]),
    # row counts: 1, 7, rows per pass (256 / (C/8) = 32 at C = 64; 8 for the scalar kernel) +- 1, a ragged last CTA
    _bnf("bn_rows1", 1, 64, kernels=[VS, AP]),
    _bnf("bn_rows7", 7, 64, kernels=[VS, AP]),
    _bnf("bn_rows31", 31, 64, kernels=[VS, AP]),
    _bnf("bn_rows33", 33, 64, kernels=[VS, AP]),
    _bnf("bn_c24_rows7", 7, 24, kernels=[SS, AP]),
    _bnf("bn_c24_rows9", 9, 24, kernels=[SS, AP]),
    _bnf("bn_rows1000_ragged_cta", 1000, 64, relu=True, kernels=[VS, AP]),
    _bnf("bn_stem_rows", 131072, 64, relu=True, fams="EF", kernels=[VS, AP]),
    # eval; gamma / beta absent; a constant channel
    _bnf("bn_eval_res_relu", 4096, 64, train=False, res=True, relu=True, fams="EF", kernels=[VS, AP]),
    _bnf("bn_eval", 1000, 64, train=False, kernels=[VS, AP]),
    _bnf("bn_no_affine", 4096, 64, affine=False, relu=True, kernels=[VS, AP]),
    _bnf("bn_const_channel", 256, 64, const=True, fams="EF", kernels=[VS, AP]),
    # |mean| = 16, 64 and 256 std: E[x^2] - mean^2 cancels in fp32
    _bnf("bn_offset16", 8192, 64, shift=16.0, fams="F", kernels=[VS, AP]),
    _bnf("bn_offset64", 8192, 64, shift=64.0, fams="F", kernels=[VS, AP]),
    _bnf("bn_offset256", 8192, 64, shift=256.0, fams="F", kernels=[VS, AP]),
    # cluster backward: every ITER and cluster size, row counts either side of 128 S ITER (4 slices at C = 64)
    _bnb("clu_rows128_s1", 128, 64, mc=16, kernels=[clu(1, 1)]),
    _bnb("clu_rows129_s2", 129, 64, mc=16, dy_b=True, kernels=[clu(1, 2)]),
    _bnb("clu_rows256_s2", 256, 64, mc=16, relu=False, kernels=[clu(1, 2)]),
    _bnb("clu_rows257_s4", 257, 64, mc=16, dres=False, kernels=[clu(1, 4)]),
    _bnb("clu_rows1024_s8", 1024, 64, mc=16, dy_b=True, fams="EF", kernels=[clu(1, 8)]),
    _bnb("clu_rows1025_s16", 1025, 64, mc=16, kernels=[clu(1, 16)]),
    _bnb("clu_rows2048_mc8_i2", 2048, 64, mc=8, dy_b=True, kernels=[clu(2, 8)]),
    _bnb("clu_rows4096_i2", 4096, 64, mc=16, dy_b=True, fams="EF", kernels=[clu(2, 16)]),
    _bnb("clu_rows4097_i4", 4097, 64, mc=16, affine=False, kernels=[clu(4, 16)]),
    _bnb("clu_rows8192_i4", 8192, 64, mc=16, dy_b=True, kernels=[clu(4, 16)]),
    _bnb("clu_rows8193_i8", 8193, 64, mc=16, kernels=[clu(8, 16)]),
    _bnb("clu_rows16384_i8", 16384, 64, mc=16, dy_b=True, fams="EF", kernels=[clu(8, 16)]),
    _bnb("clu_rows16385_i0", 16385, 64, mc=-16, dy_b=True, kernels=[clu(0, 16)]),
    _bnb("clu_rows1100_i0_s1", 1100, 64, mc=-1, kernels=[clu(0, 1)]),
    _bnb("clu_c16", 4096, 16, mc=16, dy_b=True, kernels=[clu(2, 16)]),
    _bnb("clu_c2048_halved", 1024, 2048, mc=16, fams="EF", kernels=[clu(4, 2)]),
    # two-kernel backward: vectorised and scalar reduce (C = 24, misaligned), and C = 3080 (> 48 KB of shared memory)
    _bnb("two_c64_vec", 4096, 64, fams="EF", kernels=["bn_bwd_reduce_vec", "bn_bwd_apply"]),
    _bnb("two_c24_scalar", 1024, 24, kernels=["bn_bwd_reduce", "bn_bwd_apply"]),
    _bnb("two_c64_misaligned", 2048, 64, offset=2, relu=False, kernels=["bn_bwd_reduce", "bn_bwd_apply"]),
    _bnb("two_c3080", 64, 3080, fams="EF", kernels=["bn_bwd_reduce", "bn_bwd_apply"]),
    # stem: 3x3/2 pad 1 max-pool; the 32768 x 64 map of a 32x32 batch of 128; odd maps; dead channels (p = 0)
    _stem("stem_128x16x16", 128, 16, 16, 64, dy_b=True, fams="EF"),
    _stem("stem_odd_9x11", 6, 9, 11, 64, dy_b=True, fams="EF"),
    _stem("stem_odd_dead", 4, 7, 5, 32, dead=True),
    # LayerNorm: every ROW_DISPATCH pair, rows not a multiple of the rows per block, the scalar kernels, a residual, a
    # constant row, more rows than the backward grid's groups (264 CTAs x 32 rows at C = 64)
    _ln("ln_c64", 37, 64, (8, 1), const=True),
    _ln("ln_c128", 101, 128, (16, 1), fams="EF"),
    _ln("ln_c256_res", 77, 256, (32, 1), res=True),
    _ln("ln_c512", 65, 512, (32, 2)),
    _ln("ln_c768_res", 300, 768, (32, 3), res=True, fams="EF"),
    _ln("ln_c1024", 33, 1024, (32, 4), fams="EF"),
    _ln("ln_c64_many_rows", 9000, 64, (8, 1)),
    _ln("ln_c100_scalar", 50, 100, res=True, fams="EF"),
    _ln("ln_c64_misaligned", 40, 64, offset=1, const=True),
    _ln("ln_c36_scalar_many_rows", 3000, 36),
    # softmax: the same pairs, scale != 1, BERT's additive mask of -30000 (a fully masked row), repeated maxima
    _sm("sm_c64", 37, 64, (8, 1), scale=0.5, fams="EF"),
    _sm("sm_c128_bert_mask", 1536, 128, (16, 1), scale=0.125, mask=True, fams="EF"),
    _sm("sm_c256", 77, 256, (32, 1), scale=0.125),
    _sm("sm_c512", 65, 512, (32, 2), const=True),
    _sm("sm_c768", 30, 768, (32, 3), scale=0.5, fams="EF"),
    _sm("sm_c1024", 33, 1024, (32, 4), mask=True),
    _sm("sm_c100_scalar", 50, 100, scale=0.5, fams="EF"),
    _sm("sm_c128_misaligned", 40, 128, offset=1, mask=True),
]
CASE_IDS = [c.id for c in CASES]
assert len(set(CASE_IDS)) == len(CASE_IDS)
ROW_PAIRS = [(8, 1), (16, 1), (32, 1), (32, 2), (32, 3), (32, 4)]


def _case(cid):
    return CASES[CASE_IDS.index(cid)]


def _pow2(n):
    return n > 0 and n & (n - 1) == 0


# ------------------------------------------------------------------------------------------------ data
def _shape(shape):
    return (shape,) if isinstance(shape, int) else tuple(shape)


def _ri(shape, lo, hi, g):
    shape = _shape(shape)
    return torch.randint(lo, hi + 1, shape, generator=g).double()


def _pick(shape, values, g):
    v = torch.tensor(values, dtype=F64)
    return v[torch.randint(0, len(values), _shape(shape), generator=g)]


def _quarter_means(X, g, dim=0):
    """Move single elements of the integer matrix ``X`` by +-1 so that every mean along ``dim`` is a multiple of 1/4
    (``X.shape[dim]`` a multiple of 4): each column (row) gets |d| distinct elements moved, |d| <= n / 8."""
    Xt = X if dim == 0 else X.t()
    n = Xt.shape[0]
    s = Xt.sum(0)
    d = torch.round(s * 4 / n) * n / 4 - s
    rank = torch.rand(Xt.shape, generator=g).argsort(0).argsort(0)
    Xt += torch.sign(d) * (rank < d.abs()).double()
    return X


def _randn_bf16(shape, g, scale=1.0, shift=0.0):
    return (torch.randn(_shape(shape), generator=g, dtype=F64) * scale + shift).to(BF16).double()


def _dyadic(shape, g, signed=True):
    shape = _shape(shape)
    v = _pick(shape, [0.5, 0.75, 1.0, 1.5], g)
    return v * torch.where(torch.rand(shape, generator=g) < 0.5, -1.0, 1.0).double() if signed else v


def _data(cid, fam):
    c = _case(cid)
    g = torch.Generator().manual_seed(1000 + 2 * CASE_IDS.index(cid) + (fam == "F"))
    o = c.geo
    E = fam == "E"
    if c.op == "bn_fwd":
        rows, C = o["rows"], o["C"]
        if E:
            x = _ri((rows, C), -4, 4, g)
            if _pow2(rows) and rows >= 4:
                _quarter_means(x, g)
        else:
            x = _randn_bf16((rows, C), g, 1.0, o["shift"]) if o["shift"] else _randn_bf16((rows, C), g, 1.5, 0.3)
        if o["const"]:
            x[:, 3] = 1.0
            x[:, 10] = 3.0
        d = dict(x=x)
        d["res"] = (_ri((rows, C), -3, 3, g) if E else _randn_bf16((rows, C), g)) if o["res"] else None
        d["gamma"] = (_dyadic(C, g) if E else _randn_bf16(C, g).float().double()) if o["affine"] else None
        d["beta"] = (_pick(C, [-1.0, -0.5, 0.25, 0.5, 1.0], g) if E else torch.randn(C, generator=g, dtype=F64)
                     .float().double()) if o["affine"] else None
        d["rm"] = _pick(C, [-0.5, 0.0, 0.25, 1.0], g)
        d["rv"] = _pick(C, [0.5, 1.0, 2.0, 3.0], g)
        d["prefill"] = _ri(2 * C, -64, 64, g) if E else torch.zeros(2 * C, dtype=F64)
        return d
    if c.op == "bn_bwd":
        rows, C = o["rows"], o["C"]
        if E:
            x = _ri((rows, C), -2, 2, g)
            y = _ri((rows, C), -1, 1, g)
            dy_a = _ri((rows, C), -1, 1, g) if o["dy_b"] else _ri((rows, C), -2, 2, g)
            dy_b = _ri((rows, C), -1, 1, g) if o["dy_b"] else None
            mean = _ri(C, 0, 1, g)
            rstd = _pick(C, [0.5, 1.0], g)
            gamma = _dyadic(C, g) if o["affine"] else None
            pre = _ri(2 * C, -64, 64, g)
        else:
            x = _randn_bf16((rows, C), g, 1.5, 0.3)
            y = _randn_bf16((rows, C), g)
            dy_a, dy_b = _randn_bf16((rows, C), g), (_randn_bf16((rows, C), g) if o["dy_b"] else None)
            mean = x.mean(0).float().double()
            rstd = (1.0 / torch.sqrt(x.var(0, unbiased=False) + EPS)).float().double()
            gamma = (torch.rand(C, generator=g, dtype=F64) + 0.5).float().double() if o["affine"] else None
            pre = torch.randn(2 * C, generator=g, dtype=F64).float().double()
        y[torch.rand((rows, C), generator=g) < 0.15] = 0.0          # exact zeros, a third of them -0.0: masked out
        y[(y == 0) & (torch.rand((rows, C), generator=g) < 0.33)] = -0.0
        return dict(x=x, y=y, dy_a=dy_a, dy_b=dy_b, mean=mean, rstd=rstd, gamma=gamma, prefill=pre)
    if c.op == "stem":
        N, H, W, C = o["N"], o["H"], o["W"], o["C"]
        Ho, Wo = (H + 2 * o["p"] - o["k"]) // o["s"] + 1, (W + 2 * o["p"] - o["k"]) // o["s"] + 1
        if E:
            z = _ri((N * H * W, C), -3, 3, g)
            _zero_means(z, g)
            gamma = _pick(C, [0.5, 1.0, 2.0], g)                 # +-2^j: the fp32 candidate is exactly emulated
            beta = _pick(C, [-1.0, -0.5, 0.0, 0.25, 0.5], g)
            bmean, brstd = _ri(C, -1, 1, g), _pick(C, [0.5, 1.0], g)
            bgamma = _pick(C, [-1.0, -0.5, 0.5, 1.0], g)
            dy_a = _ri((N * Ho * Wo, C), -1, 1, g)
            dy_b = _ri((N * Ho * Wo, C), -1, 1, g) if o["dy_b"] else None
            pre = _ri(2 * C, -64, 64, g)
        else:
            z = _randn_bf16((N * H * W, C), g, 1.5, 0.3)
            gamma = (torch.rand(C, generator=g, dtype=F64) + 0.5).float().double()
            beta = (torch.randn(C, generator=g, dtype=F64) * 0.3).float().double()
            bmean = z.mean(0).float().double()
            brstd = (1.0 / torch.sqrt(z.var(0, unbiased=False) + EPS)).float().double()
            bgamma = gamma
            dy_a = _randn_bf16((N * Ho * Wo, C), g)
            dy_b = _randn_bf16((N * Ho * Wo, C), g) if o["dy_b"] else None
            pre = torch.randn(2 * C, generator=g, dtype=F64).float().double()
        if o["dead"]:
            beta[: C // 2] = -64.0                                 # every ReLU output of these channels is 0
        return dict(z=z, gamma=gamma, beta=beta, rm=_pick(C, [-0.5, 0.0, 0.25], g), rv=_pick(C, [0.5, 1.0, 2.0], g),
                    bmean=bmean, brstd=brstd, bgamma=bgamma, dy_a=dy_a, dy_b=dy_b, prefill=pre, Ho=Ho, Wo=Wo)
    rows, C = o["rows"], o["C"]
    if c.op == "ln":
        if E:
            x = _ri((rows, C), -3, 3, g)
            res = _ri((rows, C), -3, 3, g) if o["res"] else None
            v = x + (res if res is not None else 0.0)
            x = _quarter_means(v, g, dim=1) - (res if res is not None else 0.0)
            gamma, beta = _dyadic(C, g), _pick(C, [-1.0, -0.5, 0.0, 0.25, 0.5], g)
            dy = _ri((rows, C), -2, 2, g)
            bmean, brstd = _ri(rows, -1, 1, g), _pick(rows, [0.5, 1.0], g)
            pre = _ri(2 * C, -64, 64, g)
        else:
            x = _randn_bf16((rows, C), g, 1.5, 0.3)
            res = _randn_bf16((rows, C), g) if o["res"] else None
            gamma = (torch.rand(C, generator=g, dtype=F64) + 0.5).float().double()
            beta = (torch.randn(C, generator=g, dtype=F64) * 0.3).float().double()
            dy = _randn_bf16((rows, C), g)
            v = x + (res if res is not None else 0.0)
            bmean = v.mean(1).float().double()
            brstd = (1.0 / torch.sqrt(v.var(1, unbiased=False) + EPS)).float().double()
            pre = torch.randn(2 * C, generator=g, dtype=F64).float().double()
        if o["const"]:
            x[1] = 2.0
            if res is not None:
                res[1] = 0.0
        return dict(x=x, res=res, gamma=gamma, beta=beta, dy=dy, bmean=bmean, brstd=brstd, prefill=pre)
    # softmax: scores (with the additive mask rounded in, as the model's bf16 scores carry it); probabilities and
    # gradients for the backward
    x = _ri((rows, C), -6, 6, g) if E else _randn_bf16((rows, C), g, 3.0)
    if o["const"]:
        x[0] = 1.0
    if o["mask"]:
        keep = torch.randint(1, C + 1, (rows,), generator=g)
        keep[1] = 0                                               # one fully masked row
        keep[2] = C
        x = (x + torch.where(torch.arange(C)[None, :] < keep[:, None], 0.0, -30000.0)).to(BF16).double()
    if E:
        yb = _ri((rows, C), 0, 16, g) / 64.0                       # dyadic "probabilities": the kernel only multiplies
        dy = _ri((rows, C), -3, 3, g)
    else:
        yb = torch.softmax(_randn_bf16((rows, C), g, 2.0), 1).to(BF16).double()
        dy = _randn_bf16((rows, C), g)
    return dict(x=x, y=yb, dy=dy)


def _zero_means(z, g):
    """Move single elements of integer ``z`` by +-1 until every column sums to 0."""
    s = z.sum(0)
    rank = torch.rand(z.shape, generator=g).argsort(0).argsort(0)
    z -= torch.sign(s) * (rank < s.abs()).double()


# ------------------------------------------------------------------------------------------------ float64 reference
def _f32(t):
    return t.float().double()


def _ulp32(t):
    _, e = torch.frexp(t.abs().float())
    return torch.ldexp(torch.ones_like(t), (e.double() - 24).clamp_min(-149).long())


def _rsqrt_arg(var, eps):
    """The kernel's ``var + eps`` in fp32, var given exactly."""
    return _f32(_f32(var).float() + torch.tensor(eps, dtype=F32))


def ref_stats(x, prefill, drop=None, dup=None):
    if drop is not None:
        x = torch.cat([x[:drop], x[drop + 1:]])
    if dup is not None:
        x = torch.cat([x, x[dup:dup + 1]])
    return prefill + torch.cat([x.sum(0), (x * x).sum(0)])


def ref_bn_moments(sums, rows, unbiased=False):
    C = sums.numel() // 2
    mean = sums[:C] / rows
    var = (sums[C:] / rows - mean * mean).clamp_min(0.0)
    if unbiased and rows > 1:
        var = var * rows / (rows - 1)
    return mean, var


def ref_rstd(var, eps, eps_inside=True):
    return 1.0 / torch.sqrt(_rsqrt_arg(var, eps)) if eps_inside else 1.0 / (torch.sqrt(var) + eps)


def ref_bn_y(x, res, mean, rstd, gamma, beta, relu):
    g = gamma if gamma is not None else 1.0
    b = beta if beta is not None else 0.0
    s = g * rstd
    y = (x - mean) * s + b
    if res is not None:
        y = y + res
    w = 8 * U * ((x * s).abs() + (mean * s).abs() + abs(b) + (res.abs() if res is not None else 0.0))
    return (y.clamp_min(0.0) if relu else y), w


def ref_running(rm, rv, mean, var, rows, unbiased=True):
    ub = var * rows / (rows - 1) if unbiased and rows > 1 else var
    return (1 - MOM) * rm + MOM * mean, (1 - MOM) * rv + MOM * ub


def ref_bn_bwd(x, y, dy, mean, rstd, gamma, relu, rows, mask_ge=False):
    """-> dx, dres (= the masked gradient), sum_g, sum_g_xhat, and the terms dx is built from."""
    g = dy * ((y >= 0) if mask_ge else (y > 0)).double() if relu else dy
    xh = (x - mean) * rstd
    sg, sgx = g.sum(0), (g * xh).sum(0)
    ka = (gamma if gamma is not None else 1.0) * rstd
    kb, kc = sg / rows, sgx / rows
    dx = ka * (g - kb - xh * kc)
    return dx, g, sg, sgx, dict(ka=ka, g=g, kb=kb, xh=xh, kc=kc)


def dx_window(t, exact, absg, absgx, n, fam):
    """Window of dx = ka (g - kb - xhat kc) (BatchNorm, stem, LayerNorm): see the module docstring."""
    w = torch.zeros_like(t["g"]) if exact else 8 * U * (t["g"].abs() + t["kb"].abs() + (t["xh"] * t["kc"]).abs())
    if fam == "F":
        w = w + CHAIN * (absg + t["xh"].abs() * absgx) / n
    return t["ka"].abs() * w


def pool_ref(y, N, H, W, k, s, p, Ho, Wo, tie="first"):
    """Max-pool of the bf16 values ``y [N H W, C]``: the first tap in raster order with the strictly largest value
    (``tie="last"``: the last one).  -> (p [N Ho Wo, C], arg)."""
    C = y.shape[1]
    y4 = y.view(N, H, W, C)
    best = torch.full((N, Ho, Wo, C), -math.inf, dtype=F64)
    arg = torch.full((N, Ho, Wo, C), 255, dtype=torch.long)
    for kh in range(k):
        for kw in range(k):
            hs = torch.arange(Ho) * s - p + kh
            ws = torch.arange(Wo) * s - p + kw
            hv, wv = (hs >= 0) & (hs < H), (ws >= 0) & (ws < W)
            cand = torch.full((N, Ho, Wo, C), -math.inf, dtype=F64)
            sub = y4[:, hs.clamp(0, H - 1)][:, :, ws.clamp(0, W - 1)]
            ok = (hv[:, None] & wv[None, :])[None, :, :, None]
            cand = torch.where(ok, sub, cand)
            better = cand > best if tie == "first" else (cand >= best) & ok
            best = torch.where(better, cand, best)
            arg = torch.where(better, torch.full_like(arg, kh * k + kw), arg)
    return best.reshape(-1, C), arg.reshape(-1, C)


def stem_dense_grad(g_pool, p, arg, N, H, W, k, s, pd, Ho, Wo):
    """The dense gradient: every window's (p > 0)-masked pooled gradient added at its argmax."""
    C = g_pool.shape[1]
    gm = g_pool * (p > 0).double()
    dense = torch.zeros(N, H, W, C, dtype=F64)
    a = arg.view(N, Ho, Wo, C)
    gm = gm.view(N, Ho, Wo, C)
    for t in range(k * k):
        kh, kw = divmod(t, k)
        hs, ws = torch.arange(Ho) * s - pd + kh, torch.arange(Wo) * s - pd + kw
        sel = (a == t).double() * gm
        for i, h in enumerate(hs.tolist()):
            if 0 <= h < H:
                for j, w in enumerate(ws.tolist()):
                    if 0 <= w < W:
                        dense[:, h, w] += sel[:, i, j]
    return dense.reshape(-1, C)


def ref_ln(v, ddof=0):
    C = v.shape[1]
    mu = v.mean(1, keepdim=True)
    var = ((v - mu) ** 2).sum(1, keepdim=True) / (C - ddof)
    return mu.squeeze(1), var.squeeze(1)


def ref_ln_bwd(x, dy, gamma, mu, rs):
    C = x.shape[1]
    h = (x - mu[:, None]) * rs[:, None]
    w = dy * gamma
    s1, s2 = w.sum(1, keepdim=True) / C, (w * h).sum(1, keepdim=True) / C
    dx = rs[:, None] * (w - s1 - h * s2)
    t = dict(ka=rs[:, None].expand_as(w), g=w, kb=s1.expand_as(w), xh=h, kc=s2.expand_as(w))
    return dx, (dy * h).sum(0), dy.sum(0), t, (w.abs().sum(1, keepdim=True), (w * h).abs().sum(1, keepdim=True))


def ref_softmax(x, scale):
    t = x * scale
    m = t.max(1, keepdim=True).values
    e = torch.exp(t - m)
    p = e / e.sum(1, keepdim=True)
    a = (t.abs() + (t - m).abs())
    a = torch.where(torch.isfinite(a), a, torch.zeros_like(a))
    w = p * U * (16 + x.shape[1] + 2 * a + (p * (8 + 2 * a)).sum(1, keepdim=True))
    return p, w


def ref_softmax_bwd(y, dy, scale, fam):
    s = (y * dy).sum(1, keepdim=True)
    dx = scale * y * (dy - s)
    if fam == "E":
        return dx, torch.zeros_like(dx)
    return dx, abs(scale) * y.abs() * (8 * U * (dy.abs() + s.abs()) + CHAIN * (y * dy).abs().sum(1, keepdim=True))


# ------------------------------------------------------------------------------------------------ checks
def _frexp_grid(r):
    a = r.abs()
    _, e = torch.frexp(a)
    ulp = torch.ldexp(torch.ones_like(a), (e - 1).clamp_min(-126) - 7)
    return a / ulp, ulp


def _round_bf16(r, mode="rne"):
    q, ulp = _frexp_grid(r)
    m = {"rne": torch.round, "trunc": torch.floor, "away": lambda t: torch.floor(t + 0.5), "up": torch.ceil}[mode](q)
    return torch.sign(r) * m * ulp


def _mismatch(tag, got, ref, bad):
    idx = bad.nonzero()[:5].tolist()
    return "{}: {} of {} elements differ, first at {}: got {} want {}".format(
        tag, int(bad.sum()), bad.numel(), idx, [float(got[tuple(i)]) for i in idx], [float(ref[tuple(i)]) for i in idx])


def check_f32(tag, got, ref, w=0.0):
    """|got - ref| <= w (w = 0: equal).  Returns the worst |got - ref| / w (0 when exact)."""
    g = got.double()
    w = torch.as_tensor(w, dtype=F64, device=g.device).expand_as(g) if not torch.is_tensor(w) else w.expand_as(g)
    err = (g - ref).abs()
    bad = ~(err <= w)
    assert not bad.any(), _mismatch(tag, g, ref, bad)
    nz = w > 0
    return float((err[nz] / w[nz]).max()) if nz.any() else 0.0


def check_bf16(tag, got, ref, w=None):
    """A bf16 ``got`` is the correct rounding of some value within ``w`` of ``ref`` (w absent or 0: ``ref`` rounded
    to nearest-even).  Returns the worst distance from a value that rounds to ``got``, as a fraction of ``w``."""
    g = got.double()
    if w is None:
        want = _round_bf16(ref)
        bad = ~(g == want)
        assert not bad.any(), _mismatch(tag, g, want, bad)
        return 0.0
    w = w.expand_as(g)
    bad = ~((g >= _round_bf16(ref - w)) & (g <= _round_bf16(ref + w)))
    assert not bad.any(), _mismatch(tag, g, _round_bf16(ref), bad)
    off = g != _round_bf16(ref)
    implied = ((g - ref).abs() - 0.5 * _frexp_grid(g)[1]).clamp_min(0.0)
    nz = off & (w > 0)
    return float((implied[nz] / w[nz]).max()) if nz.any() else 0.0


def check_rstd(tag, got, var, eps, extra_rel=0.0, ulps=2):
    """``got`` within ``ulps`` fp32 ulp of ``1/sqrt(fp32(var + eps))`` (plus ``extra_rel`` relative)."""
    ref = ref_rstd(var, eps)
    return check_f32(tag, got, ref, ulps * _ulp32(ref) + extra_rel * ref)


# ------------------------------------------------------------------------------------------------ CPU: the generator
def _ties(r):
    rne = _round_bf16(r)
    return bool((_round_bf16(r, "trunc") != rne).any()) and bool((_round_bf16(r, "away") != rne).any())


def _dyadic_ok(t, bound=EXACT_BOUND):
    """Every element of ``t`` is a multiple of 2^-b and ``max |t| 2^b`` is below ``bound``: exact in fp32, and so is
    every partial sum of such elements that stays below the same bound."""
    return float(t.abs().max()) * 2.0 ** _min_bits(t) < bound


def _f32_ok(*ts):
    """Every element of every ``t`` is an fp32 value."""
    return all(torch.equal(t, _f32(t)) for t in ts)


def _min_bits(t):
    """The fractional bits ``t``'s elements need."""
    for b in range(0, 40):
        s = t * 2.0 ** b
        if torch.equal(s, s.round()):
            return b
    return 40


def test_generator_bounds_ties_and_coverage():
    """Family E data of every case, in float64 on the CPU: every sum a kernel forms is a dyadic below 2^24, the
    statistics cases have quarter means, the exact bf16 outputs include rounding ties, and the table covers each
    kernel the issue of this module lists."""
    tie_ops = set()
    for c in CASES:
        if "E" not in c.fams:
            continue
        d = _data(c.id, "E")
        o = c.geo
        if c.op == "bn_fwd":
            rows, C = o["rows"], o["C"]
            sums = ref_stats(d["x"], d["prefill"])
            assert _dyadic_ok(sums), c.id
            if _pow2(rows):
                mean, var = ref_bn_moments(sums - d["prefill"], rows)
                assert _min_bits(mean) <= 2 and _dyadic_ok(var), c.id
        elif c.op == "bn_bwd":
            dy = d["dy_a"] + (d["dy_b"] if d["dy_b"] is not None else 0.0)
            dx, dres, sg, sgx, t = ref_bn_bwd(d["x"], d["y"], dy, d["mean"], d["rstd"], d["gamma"], o["relu"], o["rows"])
            for v in (sg, sgx, sg + d["prefill"][o["C"]:], sgx + d["prefill"][: o["C"]]):
                assert _dyadic_ok(v), c.id
            if _pow2(o["rows"]):
                assert _f32_ok(t["ka"], t["kb"], t["kc"], t["xh"] * t["kc"], t["g"] - t["kb"] - t["xh"] * t["kc"], dx), c.id
                if _ties(dx):
                    tie_ops.add("bn_bwd")
        elif c.op == "stem":
            z = d["z"]
            assert bool((z.sum(0) == 0).all()) and _dyadic_ok((z * z).sum(0)), c.id
            y, _ = _stem_fwd_ref(c, d, _rstd_guess(c, d))
            N, H, W = o["N"], o["H"], o["W"]
            p, arg = pool_ref(y, N, H, W, o["k"], o["s"], o["p"], d["Ho"], d["Wo"])
            pl, argl = pool_ref(y, N, H, W, o["k"], o["s"], o["p"], d["Ho"], d["Wo"], tie="last")
            assert torch.equal(p, pl) and not torch.equal(arg, argl), c.id      # ties between taps
            if o["dead"]:
                assert bool((p[:, : o["C"] // 2] == 0).all()), c.id
            dx, _, t = _stem_bwd_ref(c, d, p, arg)
            if _pow2(N * H * W):
                assert _f32_ok(t["ka"], t["kb"], t["kc"], t["xh"] * t["kc"], t["g"] - t["kb"] - t["xh"] * t["kc"], dx), c.id
                if _ties(dx):
                    tie_ops.add("stem")
        elif c.op == "ln":
            v = d["x"] + (d["res"] if d["res"] is not None else 0.0)
            mu, var = ref_ln(v)
            assert _min_bits(mu) <= 2 and _dyadic_ok(((v - mu[:, None]) ** 2).sum(1)), c.id
            dx, dg, db, t, _ = ref_ln_bwd(d["x"], d["dy"], d["gamma"], d["bmean"], d["brstd"])
            assert _dyadic_ok(dg) and _dyadic_ok(db), c.id
            if _pow2(o["C"]):
                assert _f32_ok(t["kb"], t["kc"], t["xh"] * t["kc"], t["g"] - t["kb"] - t["xh"] * t["kc"], dx), c.id
                if _ties(dx):
                    tie_ops.add("ln")
        else:
            dx, _ = ref_softmax_bwd(d["y"], d["dy"], o["scale"], "E")
            assert _f32_ok(dx) and _dyadic_ok((d["y"] * d["dy"]).sum(1)), c.id
            if _ties(dx):
                tie_ops.add("sm")
            t = d["x"] * o["scale"]
            assert bool(((t == t.max(1, keepdim=True).values).sum(1) > 1).any()), c.id      # repeated maxima
    assert tie_ops == {"bn_bwd", "stem", "ln", "sm"}, tie_ops
    kernels = set().union(*(c.kernels for c in CASES))
    assert {clu(i, s) for i, s in [(0, 1), (0, 16), (1, 1), (1, 2), (1, 4), (1, 8), (1, 16), (2, 8), (2, 16), (4, 16),
                                   (8, 16), (4, 2)]} <= kernels
    for name in ("layernorm_fwd", "layernorm_bwd", "softmax_fwd", "softmax_bwd"):
        assert {vec(name, *lv) for lv in ROW_PAIRS} | {name} <= kernels
    bases = {k.split("<")[0].split("/")[0] for k in kernels} | {"bn_fold_eval"}
    assert _norm_globals() <= bases, sorted(_norm_globals() - bases)


def _rstd_guess(c, d):
    """The exact stem statistics' rstd, as an fp32 value (on the GPU the kernel's own save_rstd is used)."""
    rows = c.geo["N"] * c.geo["H"] * c.geo["W"]
    _, var = ref_bn_moments(torch.cat([d["z"].sum(0), (d["z"] ** 2).sum(0)]), rows)
    return _f32(ref_rstd(var, EPS))


def _stem_fwd_ref(c, d, rstd):
    """Candidates ``bf16(fp32(fma(z, gamma rstd, beta)))`` after ReLU (zero column means: shift = beta), exactly."""
    s = d["gamma"] * rstd                       # +-2^j times an fp32 value: exact
    y = _f32(d["z"] * s + d["beta"]).clamp_min(0.0)
    return y.to(BF16).double(), s


def _stem_bwd_ref(c, d, p, arg):
    o = c.geo
    N, H, W = o["N"], o["H"], o["W"]
    gp = d["dy_a"] + (d["dy_b"] if d["dy_b"] is not None else 0.0)
    dense = stem_dense_grad(gp, p, arg, N, H, W, o["k"], o["s"], o["p"], d["Ho"], d["Wo"])
    dx, _, sg, sgx, t = ref_bn_bwd(d["z"], torch.ones_like(dense), dense, d["bmean"], d["brstd"], d["bgamma"], False,
                                   N * H * W)
    return dx, (sg, sgx, dense), t


def test_checks_reject_plausible_mistakes():
    """On the CPU, in float64: each mistake below makes a float64 'kernel output' that the checks of this module
    reject, on the case data they run on the GPU."""
    c = _case("bn_c64_res_relu")
    d = _data(c.id, "E")
    x, rows = d["x"], c.geo["rows"]
    sums = ref_stats(x, d["prefill"])
    for bad in (ref_stats(x, d["prefill"], drop=rows - 1), ref_stats(x, d["prefill"], drop=17),
                ref_stats(x, d["prefill"], dup=rows - 1)):
        with pytest.raises(AssertionError):                 # a dropped or a duplicated row
            check_f32("sums", bad, sums)
    mean, var = ref_bn_moments(sums - d["prefill"], rows)
    rstd = _f32(ref_rstd(var, EPS))
    check_rstd("rstd", rstd, var, EPS)
    with pytest.raises(AssertionError):                     # eps outside the square root
        check_rstd("rstd", _f32(ref_rstd(var, EPS, eps_inside=False)), var, EPS)
    with pytest.raises(AssertionError):                     # the unbiased variance normalises
        check_rstd("rstd", _f32(ref_rstd(var * rows / (rows - 1), EPS)), var, EPS)
    rm, rv = ref_running(d["rm"], d["rv"], mean, var, rows)
    _, rv_biased = ref_running(d["rm"], d["rv"], mean, var, rows, unbiased=False)
    with pytest.raises(AssertionError):                     # biased variance in the running statistics
        check_f32("running_var", rv_biased, rv, _running_window(rm, rv, d, mean, var, rows)[1])
    y, w = ref_bn_y(x, d["res"], mean, rstd, d["gamma"], d["beta"], True)
    for bad in (ref_stats(x, d["prefill"], drop=rows - 1), ref_stats(x, d["prefill"], dup=3)):
        m2, v2 = ref_bn_moments(bad - d["prefill"], rows)
        y2, _ = ref_bn_y(x, d["res"], m2, _f32(ref_rstd(v2, EPS)), d["gamma"], d["beta"], True)
        with pytest.raises(AssertionError):                 # ... and y from the statistics of such a sum
            check_bf16("y", y2.to(BF16), y, w)
    # backward: a dropped / duplicated row in the sums, an ignored dy_b, a ReLU mask of y >= 0, truncating rounding
    c = _case("clu_rows4096_i2")
    d = _data(c.id, "E")
    rows = c.geo["rows"]
    dy = d["dy_a"] + d["dy_b"]
    dx, dres, sg, sgx, _ = ref_bn_bwd(d["x"], d["y"], dy, d["mean"], d["rstd"], d["gamma"], True, rows)
    check_bf16("dx", dx.to(BF16), dx)
    t = ref_bn_bwd(d["x"], d["y"], dy, d["mean"], d["rstd"], d["gamma"], True, rows)[4]
    for sl in (slice(0, rows - 1), torch.cat([torch.arange(rows), torch.tensor([5])])):
        _, _, sg2, sgx2, _ = ref_bn_bwd(d["x"][sl], d["y"][sl], dy[sl], d["mean"], d["rstd"], d["gamma"], True, rows)
        with pytest.raises(AssertionError):
            check_f32("dgamma", sgx2, sgx)
        dx2 = t["ka"] * (t["g"] - sg2 / rows - t["xh"] * sgx2 / rows)
        with pytest.raises(AssertionError):
            check_bf16("dx", _round_bf16(dx2), dx)
    dx_a, dres_a, _, _, _ = ref_bn_bwd(d["x"], d["y"], d["dy_a"], d["mean"], d["rstd"], d["gamma"], True, rows)
    with pytest.raises(AssertionError):
        check_bf16("dx ignoring dy_b", _round_bf16(dx_a), dx)
    dx_ge, dres_ge, _, _, _ = ref_bn_bwd(d["x"], d["y"], dy, d["mean"], d["rstd"], d["gamma"], True, rows,
                                         mask_ge=True)
    with pytest.raises(AssertionError):
        check_bf16("dres with y >= 0", dres_ge, dres)
    with pytest.raises(AssertionError):
        check_bf16("dx with y >= 0", _round_bf16(dx_ge), dx)
    for mode in ("trunc", "away"):
        with pytest.raises(AssertionError):
            check_bf16(mode, _round_bf16(dx, mode), dx)
    # the stem's tie rule: the last of the equal maxima instead of the first
    c = _case("stem_odd_9x11")
    d = _data(c.id, "E")
    o = c.geo
    y, _ = _stem_fwd_ref(c, d, _rstd_guess(c, d))
    args = [pool_ref(y, o["N"], o["H"], o["W"], o["k"], o["s"], o["p"], d["Ho"], d["Wo"], tie=t)[1]
            for t in ("first", "last")]
    with pytest.raises(AssertionError):
        check_f32("argmax", args[1].double(), args[0].double())
    # the LayerNorm variance divided by C - 1
    c = _case("ln_c1024")
    d = _data(c.id, "E")
    v = d["x"]
    mu, var = ref_ln(v)
    _, var1 = ref_ln(v, ddof=1)
    with pytest.raises(AssertionError):
        check_rstd("ln rstd", _f32(ref_rstd(var1, EPS)), var, EPS)


def _running_window(rm, rv, d, mean, var, rows, dvar=0.0):
    wm = 4 * U * ((1 - MOM) * d["rm"].abs() + MOM * mean.abs())
    f = rows / (rows - 1) if rows > 1 else 1.0
    wv = 4 * U * (1 - MOM) * d["rv"].abs() + MOM * (6 * U * var * f + dvar * f)
    return wm, wv


# ------------------------------------------------------------------------------------------------ GPU
def _guarded(shape, dtype, dev, *, offset=0, tail=67, prefill=None):
    """``shape`` view at element ``offset`` of a buffer with a tail, every element holding the NaN sentinel; returns
    ``(view, check)``: ``check(tag)`` asserts the guard elements kept their bits."""
    n = math.prod(shape)
    idt, bits = SENTINEL[dtype]
    buf = torch.full((offset + n + tail,), bits, dtype=idt, device=dev)
    view = buf[offset: offset + n].view(dtype).view(shape)
    if prefill is not None:
        view.copy_(prefill)
    guard = torch.ones_like(buf, dtype=torch.bool)
    guard[offset: offset + n] = False

    def check(tag):
        changed = int((buf[guard] != bits).sum())
        assert changed == 0, "{}: {} guard elements overwritten".format(tag, changed)
    return view, check


def _placed(t, dtype, dev, offset=0):
    """``t`` copied to element ``offset`` of a fresh buffer (offset 0: an aligned tensor)."""
    if t is None:
        return None
    buf = torch.zeros(offset + t.numel() + 8, dtype=dtype, device=dev)
    v = buf[offset: offset + t.numel()].view(t.shape)
    v.copy_(t.to(dtype))
    return v


@pytest.fixture(scope="module")
def C_():
    from baton_b200.ops import load
    return load()


def _report(tag, ratios):
    print("{}: worst error / window: {}".format(tag, ", ".join("{} {:.3g}".format(k, v) for k, v in ratios.items())))


def _run_bn_fwd(c, d, fam, C_, dev):
    o = c.geo
    rows, C = o["rows"], o["C"]
    checks, out = [], {}
    xs = _placed(d["x"], BF16, dev, o["offset"])
    sums, chk = _guarded((2 * C,), F32, dev, prefill=d["prefill"].float())
    checks.append(chk)
    C_.bn_stats(xs, sums, rows, C)
    out["sums"] = sums
    sums_apply = (sums - d["prefill"].float().to(dev)).contiguous()
    x = _placed(d["x"], BF16, dev)
    res = _placed(d["res"], BF16, dev)
    y, chk = _guarded((rows, C), BF16, dev)
    checks.append(chk)
    sm, chk_m = _guarded((C,), F32, dev)
    sr, chk_r = _guarded((C,), F32, dev)
    rm, chk_rm = _guarded((C,), F32, dev, prefill=d["rm"].float())
    rv, chk_rv = _guarded((C,), F32, dev, prefill=d["rv"].float())
    nbt, chk_n = _guarded((1,), torch.int64, dev, prefill=torch.tensor([41]))
    checks += [chk_m, chk_r, chk_rm, chk_rv, chk_n]
    gamma = d["gamma"].float().to(dev) if d["gamma"] is not None else None
    beta = d["beta"].float().to(dev) if d["beta"] is not None else None
    C_.bn_apply(x, res, y, sums_apply, gamma, beta, rm, rv, sm, sr, nbt.view(()), rows, C, EPS, MOM, o["relu"],
                o["train"])
    out.update(y=y, save_mean=sm, save_rstd=sr, rm=rm, rv=rv, nbt=nbt, sums_apply=sums_apply)
    return out, checks


def _check_bn_fwd(c, d, fam, out, dev):
    o = c.geo
    rows, C = o["rows"], o["C"]
    cpu = {k: (v.cpu() if torch.is_tensor(v) else v) for k, v in out.items()}
    r = {}
    x = d["x"]
    ref = ref_stats(x, d["prefill"])
    absx = torch.cat([x.abs().sum(0), (x * x).sum(0)])
    r["sums"] = check_f32(c.id + " sums", cpu["sums"], ref, 0.0 if fam == "E" else CHAIN * absx)
    if not o["train"]:
        assert bool(torch.isnan(cpu["save_mean"]).all() and torch.isnan(cpu["save_rstd"]).all()), c.id
        assert torch.equal(cpu["rm"].double(), d["rm"]) and torch.equal(cpu["rv"].double(), d["rv"]), c.id
        assert int(cpu["nbt"]) == 41, c.id
        mean, rstd_ref = d["rm"], ref_rstd(d["rv"], EPS)
        y, w = ref_bn_y(x, d["res"], mean, rstd_ref, d["gamma"], d["beta"], o["relu"])
        g = d["gamma"] if d["gamma"] is not None else 1.0
        w = w + 2.0 ** -21 * ((x - mean) * g * rstd_ref).abs()            # rsqrtf's 2 ulp
        r["y"] = check_bf16(c.id + " y", cpu["y"], y, w)
        return r
    assert int(cpu["nbt"]) == 42, c.id
    s = _f32(cpu["sums_apply"])
    mean_ref, var_ref = ref_bn_moments(s, rows)
    exact = fam == "E" and _pow2(rows)
    r["save_mean"] = check_f32(c.id + " save_mean", cpu["save_mean"], mean_ref, 0.0 if exact else 4 * U * mean_ref.abs())
    ex2 = s[C:] / rows
    dvar = torch.zeros(C, dtype=F64) if exact else 6 * U * (ex2 + mean_ref ** 2)
    r["save_rstd"] = check_rstd(c.id + " save_rstd", cpu["save_rstd"], var_ref, EPS,
                                extra_rel=0.5 * dvar / _rsqrt_arg(var_ref, EPS), ulps=2 if exact else 3)
    rstd_k = _f32(cpu["save_rstd"])
    assert bool(torch.isfinite(rstd_k).all()) and bool((rstd_k <= (1 + 2 ** -21) / math.sqrt(EPS)).all()), c.id
    if o["shift"]:                        # end to end against the float64 statistics of the data: report only
        m64, v64 = x.mean(0), x.var(0, unbiased=False)
        e = ((rstd_k - 1.0 / torch.sqrt(v64 + EPS)).abs() * torch.sqrt(v64 + EPS)).max()
        bound = 0.5 * (CHAIN + 6 * U) * float(((x * x).mean(0) / (v64 + EPS)).max()) + 2 ** -22
        print("{}: |mean| / std = {:.0f}, rstd relative error {:.3g} (2^{:.1f}), bound {:.3g}".format(
            c.id, float((m64.abs() / v64.sqrt()).min()), float(e), math.log2(float(e)) if e > 0 else -math.inf, bound))
        assert float(e) <= bound, c.id
    mean_k = _f32(cpu["save_mean"])
    y, w = ref_bn_y(x, d["res"], mean_k, rstd_k, d["gamma"], d["beta"], o["relu"])
    r["y"] = check_bf16(c.id + " y", cpu["y"], y, w)
    if o["const"]:
        assert not bool(torch.isnan(cpu["y"].float()).any()), c.id
        if d["beta"] is not None and fam == "E":
            for ch in (3, 10):
                assert bool((cpu["y"][:, ch].double() == _round_bf16(d["beta"][ch]).clamp_min(0.0 if o["relu"] else
                                                                                               -math.inf)).all()), c.id
    rm, rv = ref_running(d["rm"], d["rv"], mean_ref, var_ref, rows)
    wm, wv = _running_window(rm, rv, d, mean_ref, var_ref, rows, dvar)
    r["running_mean"] = check_f32(c.id + " running_mean", cpu["rm"], rm, wm + MOM * (0.0 if exact else 4 * U *
                                                                                      mean_ref.abs()))
    r["running_var"] = check_f32(c.id + " running_var", cpu["rv"], rv, wv)
    return r


def _run_bn_bwd(c, d, fam, C_, dev):
    o = c.geo
    rows, C, off = o["rows"], o["C"], o["offset"]
    checks, out = [], {}
    gamma = d["gamma"].float().to(dev) if d["gamma"] is not None else None
    mean, rstd = d["mean"].float().to(dev), d["rstd"].float().to(dev)
    dx, chk = _guarded((rows, C), BF16, dev)
    checks.append(chk)
    dres = None
    if o["dres"]:
        dres, chk = _guarded((rows, C), BF16, dev)
        checks.append(chk)
    dg, chk_g = _guarded((C,), F32, dev, prefill=d["prefill"][:C].float())
    db, chk_b = _guarded((C,), F32, dev, prefill=d["prefill"][C:].float())
    checks += [chk_g, chk_b]
    x, y, dy_a = (_placed(d[k], BF16, dev) for k in ("x", "y", "dy_a"))
    if o["mc"] is not None:
        ok = C_.bn_bwd_cluster(x, y, dy_a, _placed(d["dy_b"], BF16, dev), dx, dres, gamma, mean, rstd, dg, db, rows, C,
                               o["relu"], o["mc"])
        assert ok, c.id
    else:
        sums, chk = _guarded((2 * C,), F32, dev, prefill=torch.zeros(2 * C))
        checks.append(chk)
        C_.bn_bwd_reduce(*(_placed(d[k], BF16, dev, off) for k in ("x", "y", "dy_a")), mean, rstd, sums, rows, C,
                         o["relu"])
        C_.bn_bwd_apply(x, y, dy_a, dx, dres, gamma, mean, rstd, sums, dg, db, rows, C, o["relu"])
        out["sums"] = sums
    out.update(dx=dx, dres=dres, dgamma=dg, dbeta=db)
    return out, checks


def _check_bn_bwd(c, d, fam, out, dev):
    o = c.geo
    rows, C = o["rows"], o["C"]
    cpu = {k: (v.cpu() if torch.is_tensor(v) else v) for k, v in out.items()}
    dy = d["dy_a"] + (d["dy_b"] if d["dy_b"] is not None else 0.0)
    dx, dres, sg, sgx, t = ref_bn_bwd(d["x"], d["y"], dy, d["mean"], d["rstd"], d["gamma"], o["relu"], rows)
    absg, absgx = t["g"].abs().sum(0), (t["g"] * t["xh"]).abs().sum(0)
    r = {}
    ch = (lambda a: 0.0) if fam == "E" else (lambda a: CHAIN * a)
    pre = d["prefill"]
    r["dgamma"] = check_f32(c.id + " dgamma", cpu["dgamma"], pre[:C] + sgx, ch(absgx) + (0 if fam == "E" else
                                                                                       U * (pre[:C] + sgx).abs()))
    r["dbeta"] = check_f32(c.id + " dbeta", cpu["dbeta"], pre[C:] + sg, ch(absg) + (0 if fam == "E" else
                                                                                   U * (pre[C:] + sg).abs()))
    if "sums" in cpu:
        r["sums"] = check_f32(c.id + " sums", cpu["sums"], torch.cat([sg, sgx]), ch(torch.cat([absg, absgx])))
    if o["dres"]:
        r["dres"] = check_bf16(c.id + " dres", cpu["dres"], dres)
    exact = fam == "E" and _pow2(rows)
    w = dx_window(t, exact, absg, absgx, rows, fam)
    r["dx"] = check_bf16(c.id + " dx", cpu["dx"], dx, None if exact else w)
    return r


def _run_stem(c, d, fam, C_, dev):
    o = c.geo
    N, H, W, C, k, s, p = (o[n] for n in ("N", "H", "W", "C", "k", "s", "p"))
    Ho, Wo = d["Ho"], d["Wo"]
    checks, out = [], {}
    z = _placed(d["z"], BF16, dev)
    zs = z.float()
    sums = torch.cat([zs.sum(0), (zs * zs).sum(0)]) if fam == "F" else \
        torch.cat([d["z"].sum(0), (d["z"] ** 2).sum(0)]).float().to(dev)
    pp, chk_p = _guarded((N * Ho * Wo, C), BF16, dev)
    arg, chk_a = _guarded((N * Ho * Wo, C), torch.uint8, dev)
    sm, chk_m = _guarded((C,), F32, dev)
    sr, chk_r = _guarded((C,), F32, dev)
    rm, chk_rm = _guarded((C,), F32, dev, prefill=d["rm"].float())
    rv, chk_rv = _guarded((C,), F32, dev, prefill=d["rv"].float())
    nbt, chk_n = _guarded((1,), torch.int64, dev, prefill=torch.tensor([41]))
    checks += [chk_p, chk_a, chk_m, chk_r, chk_rm, chk_rv, chk_n]
    assert C_.bn_relu_maxpool(z, pp, arg, sums, d["gamma"].float().to(dev), d["beta"].float().to(dev), rm, rv, sm, sr,
                              nbt.view(()), N, H, W, C, k, s, p, Ho, Wo, EPS, MOM)
    out.update(p=pp, arg=arg, save_mean=sm, save_rstd=sr, rm=rm, rv=rv, nbt=nbt, sums=sums)
    # backward, from the reference forward at the backward's own (mean, rstd, gamma)
    yb = ((d["z"] - d["bmean"]) * d["brstd"] * d["bgamma"] + d["beta"]).clamp_min(0.0).to(BF16).double()
    pb, ab = pool_ref(yb, N, H, W, k, s, p, Ho, Wo)
    dz, chk = _guarded((N * H * W, C), BF16, dev)
    dg, chk_g = _guarded((C,), F32, dev, prefill=d["prefill"][:C].float())
    db, chk_b = _guarded((C,), F32, dev, prefill=d["prefill"][C:].float())
    scratch = torch.zeros(2 * C, device=dev)
    checks += [chk, chk_g, chk_b]
    assert C_.bn_maxpool_bwd(z, _placed(pb, BF16, dev), ab.to(torch.uint8).to(dev), _placed(d["dy_a"], BF16, dev),
                             _placed(d["dy_b"], BF16, dev), dz, d["bgamma"].float().to(dev), d["bmean"].float().to(dev),
                             d["brstd"].float().to(dev), scratch, dg, db, N, H, W, C, k, s, p, Ho, Wo)
    out.update(dz=dz, dgamma=dg, dbeta=db, pb=pb, ab=ab)
    return out, checks


def _check_stem(c, d, fam, out, dev):
    o = c.geo
    N, H, W, C, k, s, p = (o[n] for n in ("N", "H", "W", "C", "k", "s", "p"))
    Ho, Wo, rows = d["Ho"], d["Wo"], o["N"] * o["H"] * o["W"]
    cpu = {kk: (v.cpu() if torch.is_tensor(v) else v) for kk, v in out.items()}
    r = {}
    assert int(cpu["nbt"]) == 42, c.id
    sums = _f32(cpu["sums"])
    mean_ref, var_ref = ref_bn_moments(sums, rows)
    exact = fam == "E" and _pow2(rows)
    r["save_mean"] = check_f32(c.id + " save_mean", cpu["save_mean"], mean_ref,
                               0.0 if fam == "E" else 4 * U * mean_ref.abs())
    dvar = torch.zeros(C, dtype=F64) if exact else 6 * U * (sums[C:] / rows + mean_ref ** 2)
    r["save_rstd"] = check_rstd(c.id + " save_rstd", cpu["save_rstd"], var_ref, EPS,
                                extra_rel=0.5 * dvar / _rsqrt_arg(var_ref, EPS), ulps=2 if exact else 3)
    rm, rv = ref_running(d["rm"], d["rv"], mean_ref, var_ref, rows)
    wm, wv = _running_window(rm, rv, d, mean_ref, var_ref, rows, dvar)
    r["running_mean"] = check_f32(c.id + " running_mean", cpu["rm"], rm, wm + 4 * U * MOM * mean_ref.abs())
    r["running_var"] = check_f32(c.id + " running_var", cpu["rv"], rv, wv)
    rstd_k, mean_k = _f32(cpu["save_rstd"]), _f32(cpu["save_mean"])
    if fam == "E":
        y, _ = _stem_fwd_ref(c, d, rstd_k)
        pr, ar = pool_ref(y, N, H, W, k, s, p, Ho, Wo)
        check_bf16(c.id + " p", cpu["p"], pr)
        check_f32(c.id + " argmax", cpu["arg"].double(), ar.double())
    else:
        y, w = ref_bn_y(d["z"], None, mean_k, rstd_k, d["gamma"], d["beta"], True)
        pr, _ = pool_ref(y, N, H, W, k, s, p, Ho, Wo)
        pw, _ = pool_ref(w, N, H, W, k, s, p, Ho, Wo)
        r["p"] = check_bf16(c.id + " p", cpu["p"], pr, pw)
        # the chosen tap's value rounds to p within its window
        a = cpu["arg"].long().view(N, Ho, Wo, C)
        hs = (torch.arange(Ho) * s - p)[None, :, None, None] + a // k
        ws = (torch.arange(Wo) * s - p)[None, None, :, None] + a % k
        assert bool(((hs >= 0) & (hs < H) & (ws >= 0) & (ws < W)).all()), c.id
        idx = ((torch.arange(N)[:, None, None, None] * H + hs) * W + ws).reshape(-1, C)
        ya, wa = torch.gather(y, 0, idx), torch.gather(w, 0, idx)
        check_bf16(c.id + " p at argmax", cpu["p"], ya, wa + pw)
    dx, (sg, sgx, dense), t = _stem_bwd_ref(c, d, cpu["pb"], cpu["ab"])
    absg, absgx = t["g"].abs().sum(0), (t["g"] * t["xh"]).abs().sum(0)
    pre = d["prefill"]
    ch = (lambda a_: 0.0) if fam == "E" else (lambda a_: CHAIN * a_)
    r["dgamma"] = check_f32(c.id + " dgamma", cpu["dgamma"], pre[:C] + sgx,
                            ch(absgx) + (0 if fam == "E" else U * (pre[:C] + sgx).abs()))
    r["dbeta"] = check_f32(c.id + " dbeta", cpu["dbeta"], pre[C:] + sg,
                           ch(absg) + (0 if fam == "E" else U * (pre[C:] + sg).abs()))
    w = dx_window(t, exact, absg, absgx, rows, fam)
    r["dz"] = check_bf16(c.id + " dz", cpu["dz"], dx, None if exact else w)
    return r


def _run_ln(c, d, fam, C_, dev):
    o = c.geo
    rows, C, off = o["rows"], o["C"], o["offset"]
    checks, out = [], {}
    y, chk = _guarded((rows, C), BF16, dev, offset=off)
    mean, chk_m = _guarded((rows,), F32, dev)
    rstd, chk_r = _guarded((rows,), F32, dev)
    checks += [chk, chk_m, chk_r]
    gamma, beta = d["gamma"].float().to(dev), d["beta"].float().to(dev)
    C_.layernorm_fwd(_placed(d["x"], BF16, dev, off), _placed(d["res"], BF16, dev, off), y, gamma, beta, mean, rstd,
                     rows, C, EPS)
    dx, chk = _guarded((rows, C), BF16, dev, offset=off)
    dg, chk_g = _guarded((C,), F32, dev, prefill=d["prefill"][:C].float())
    db, chk_b = _guarded((C,), F32, dev, prefill=d["prefill"][C:].float())
    checks += [chk, chk_g, chk_b]
    C_.layernorm_bwd(_placed(d["x"], BF16, dev, off), _placed(d["dy"], BF16, dev, off), dx, gamma,
                     d["bmean"].float().to(dev), d["brstd"].float().to(dev), dg, db, rows, C)
    out.update(y=y, mean=mean, rstd=rstd, dx=dx, dgamma=dg, dbeta=db)
    return out, checks


def _check_ln(c, d, fam, out, dev):
    o = c.geo
    rows, C = o["rows"], o["C"]
    cpu = {k: v.cpu() for k, v in out.items()}
    r = {}
    v = d["x"] + (d["res"] if d["res"] is not None else 0.0)
    mu, var = ref_ln(v)
    exact = fam == "E" and _pow2(C)
    sabs = v.abs().sum(1) / C
    r["mean"] = check_f32(c.id + " mean", cpu["mean"], mu,
                          0.0 if exact else 4 * U * mu.abs() + (CHAIN * sabs if fam == "F" else 0.0))
    dvar = 0.0 if fam == "E" else CHAIN * (((v - mu[:, None]) ** 2).sum(1) / C + sabs ** 2 * 4 * U)
    r["rstd"] = check_rstd(c.id + " rstd", cpu["rstd"], var, EPS, extra_rel=0.5 * dvar / _rsqrt_arg(var, EPS),
                           ulps=2 if exact else 3)
    mk, rk = _f32(cpu["mean"])[:, None], _f32(cpu["rstd"])[:, None]
    y = (v - mk) * rk * d["gamma"] + d["beta"]
    w = 8 * U * ((v * rk * d["gamma"]).abs() + (mk * rk * d["gamma"]).abs() + d["beta"].abs())
    r["y"] = check_bf16(c.id + " y", cpu["y"], y, w)
    if o["const"]:
        assert torch.equal(cpu["y"][1].double(), _round_bf16(d["beta"])), c.id
    dx, dg, db, t, (aw, awh) = ref_ln_bwd(d["x"], d["dy"], d["gamma"], d["bmean"], d["brstd"])
    h = t["xh"]
    pre = d["prefill"]
    r["dgamma"] = check_f32(c.id + " dgamma", cpu["dgamma"], pre[:C] + dg,
                            0.0 if fam == "E" else CHAIN * (d["dy"] * h).abs().sum(0) + U * (pre[:C] + dg).abs())
    r["dbeta"] = check_f32(c.id + " dbeta", cpu["dbeta"], pre[C:] + db,
                           0.0 if fam == "E" else CHAIN * d["dy"].abs().sum(0) + U * (pre[C:] + db).abs())
    w = dx_window(t, exact, aw, awh, C, fam)
    r["dx"] = check_bf16(c.id + " dx", cpu["dx"], dx, None if exact else w)
    return r


def _run_sm(c, d, fam, C_, dev):
    o = c.geo
    rows, C, off = o["rows"], o["C"], o["offset"]
    y, chk = _guarded((rows, C), BF16, dev, offset=off)
    C_.softmax_fwd(_placed(d["x"], BF16, dev, off), y, rows, C, o["scale"])
    dx, chk2 = _guarded((rows, C), BF16, dev, offset=off)
    C_.softmax_bwd(_placed(d["y"], BF16, dev, off), _placed(d["dy"], BF16, dev, off), dx, rows, C, o["scale"])
    return dict(y=y, dx=dx), [chk, chk2]


def _check_sm(c, d, fam, out, dev):
    o = c.geo
    cpu = {k: v.cpu() for k, v in out.items()}
    r = {}
    p, w = ref_softmax(d["x"], o["scale"])
    r["p"] = check_bf16(c.id + " p", cpu["y"], p, w)
    if o["mask"]:
        masked = d["x"] < -20000
        full = masked.all(1)
        assert bool((cpu["y"].double()[masked & ~full[:, None]] == 0).all()), c.id
        assert bool(full.any()) and bool((cpu["y"].double()[full] == _round_bf16(torch.tensor(1.0 / o["C"]))).all())
    dx, wdx = ref_softmax_bwd(d["y"], d["dy"], o["scale"], fam)
    r["dx"] = check_bf16(c.id + " dx", cpu["dx"], dx, None if fam == "E" else wdx)
    return r


_RUN = {"bn_fwd": (_run_bn_fwd, _check_bn_fwd), "bn_bwd": (_run_bn_bwd, _check_bn_bwd), "stem": (_run_stem, _check_stem),
        "ln": (_run_ln, _check_ln), "sm": (_run_sm, _check_sm)}


def _run_and_check(c, fam, C_):
    dev = torch.device("cuda:0")
    d = _data(c.id, fam)
    run, chk = _RUN[c.op]
    out, guards = run(c, d, fam, C_, dev)
    torch.cuda.synchronize()
    r = chk(c, d, fam, out, dev)
    for g in guards:
        g(c.id)
    return r


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=CASE_IDS)
def test_exact_integer_operands(case, C_):
    if "E" not in case.fams:
        pytest.skip("full-mantissa case")
    _run_and_check(case, "E", C_)


@pytest.mark.gpu
@pytest.mark.parametrize("case", [c for c in CASES if "F" in c.fams], ids=[c.id for c in CASES if "F" in c.fams])
def test_full_mantissa_operands(case, C_):
    _report(case.id + " (F)", _run_and_check(case, "F", C_))


@pytest.mark.gpu
def test_row_kernels_reject_rows_over_1024(C_):
    """C = 1032 is beyond the 32 elements per lane the row kernels hold: every entry point raises."""
    dev = torch.device("cuda:0")
    rows, C = 4, 1032
    x = torch.zeros(rows, C, dtype=BF16, device=dev)
    f = torch.zeros(C, device=dev)
    r = torch.zeros(rows, device=dev)
    calls = [lambda: C_.layernorm_fwd(x, None, x.clone(), f, f, r, r.clone(), rows, C, EPS),
             lambda: C_.layernorm_bwd(x, x, x.clone(), f, r, r, f.clone(), f.clone(), rows, C),
             lambda: C_.softmax_fwd(x, x.clone(), rows, C, 1.0),
             lambda: C_.softmax_bwd(x, x, x.clone(), rows, C, 1.0)]
    for call in calls:
        with pytest.raises(RuntimeError, match="failed with code -2"):
            call()
    torch.cuda.synchronize()


_KERNEL = re.compile(r"b200::(\w+)_kernel(?:<([^>]*)>)?\(")


def _kernel_key(name, grid_y=None):
    m = _KERNEL.search(name)
    if m is None:
        return None
    args = ",".join(a.strip() for a in (m.group(2) or "").split(",")) if m.group(2) else None
    key = m.group(1) + ("<{}>".format(args) if args else "")
    if m.group(1) == "bn_bwd_cluster":
        key += "/S{}".format(grid_y)
    return key


def test_kernel_key_parses_demangled_names():
    assert _kernel_key("void b200::layernorm_fwd_vec_kernel<32, 3>(__nv_bfloat16 const*, ...)") == \
        vec("layernorm_fwd", 32, 3)
    assert _kernel_key("void b200::bn_bwd_cluster_kernel<4>(uint4 const*, ...)", 16) == clu(4, 16)
    assert _kernel_key("b200::bn_stats_vec_kernel(uint4 const*, float*, long long, int, int)") == VS
    assert _kernel_key("b200::bn_fold_eval_kernel(float const*, long long const*, float*)") == "bn_fold_eval"


def _norm_globals():
    src = open(os.path.join(os.path.dirname(__file__), "..", "baton_b200", "csrc", "norm.cu")).read()
    return set(re.findall(r"__global__ void __launch_bounds__\(\d+\)\s+(\w+)_kernel\(", src))


@pytest.mark.gpu
def test_case_table_reaches_every_kernel_instantiation(C_):
    """Every case's first family under torch.profiler: every kernel the table names appears (the cluster kernel with
    its grid's cluster size), and the names cover every ``__global__`` of norm.cu and every instantiation dispatch can
    pick.  So a dispatch change that moves cases onto another kernel fails here."""
    from torch.profiler import ProfilerActivity, profile
    dev = torch.device("cuda:0")
    want = set().union(*(c.kernels for c in CASES)) | {"bn_fold_eval"}
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for c in CASES:
            fam = c.fams[0]
            _RUN[c.op][0](c, _data(c.id, fam), fam, C_, dev)
        arena = torch.tensor([1.0, 2.0, 0.5, 4.0] * 8, device=dev)
        table = torch.tensor([[0, 8, 16, 24, 0, 8, int(torch.tensor(EPS, dtype=F32).view(torch.int32))]],
                             dtype=torch.int64, device=dev)
        C_.bn_fold_eval(arena, table, torch.zeros(16, device=dev))
        torch.cuda.synchronize()
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "trace.json")
        prof.export_chrome_trace(path)
        events = json.load(open(path))["traceEvents"]
    seen = {_kernel_key(e["name"], (e.get("args", {}).get("grid") or [0, 0])[1]) for e in events
            if e.get("cat") == "kernel"} - {None}
    assert want <= seen, sorted(want - seen)
    for name in ("layernorm_fwd", "layernorm_bwd", "softmax_fwd", "softmax_bwd"):
        assert {vec(name, *lv) for lv in ROW_PAIRS} <= want
    assert {"bn_bwd_cluster<{}>".format(i) for i in (0, 1, 2, 4, 8)} <= {k.split("/")[0] for k in want}
    assert {"S{}".format(s) for s in (1, 2, 4, 8, 16)} <= {k.split("/")[1] for k in want if "/" in k}
