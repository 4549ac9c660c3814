"""The fused attention kernels (csrc/attention.cu) and the multi-kernel attention path (ops/nn.py ``_AttnFn``) against
float64, element by element.  Every case is built on the CPU from a seeded generator.  The fused kernels are called
through their extension entry points (``attention_fwd``, ``attention_bwd`` and the ``_drop_`` forms); the multi-kernel
path through ``bnn.attention`` with autograd.  The references follow each kernel's documented formula in float64; they
never call a kernel or PyTorch's bf16 path.  Dropout uses p = 0.5 (s = 2, exact) and the host mask of
``data/dropout.dropout_keep``; element i of the mask is the index into ``probs [B*H*S, S]``.

Family E (exact), fused forward.  ``scale = fp32(ln 2)``, so the kernel's ``scale_log2e = scale * fp32(log2 e)`` is
exactly 1.0 (asserted in fp32 below).  Q and K are sparse small integers, so the scores x are integers and
``P~ = 2^(x - max)`` is a power of two; bf16(P~) is exact even if ``ex2.approx`` is a few ulp off.  V is a small
integer.  The generator asserts ``x - max >= -16`` and ``sum_k P~_k |v_k| 2^16 < 2^24``, so the row sum and
``O~ = P~ V`` are exact in fp32 in any order.  Only ``1/sum`` (an approximate reciprocal under ``--use_fast_math``)
and the final products round: ``out`` and ``probs`` must be the nearest-even bf16 of the float64 value, except in a
band of relative half-width ``BAND = 2^-20`` around a rounding boundary, where either neighbour is accepted.  The
generator also asserts that every key position 0..127 is some row's dominant key with P >= 1/4, and that every
(16-byte chunk, r & 7) pair of the 128-byte swizzle carries such a key.

Family E, fused backward.  ``attention_bwd`` reads ``probs`` as an input, so it gets a crafted dyadic P (multiples of
1/128 up to 1/4); qkv and dO are small integers and ``scale = 0.125``.  dV, dP and delta are then exact in fp32, the
kernel's one intermediate rounding is ``dS = RNE_bf16(P (dP - delta))``, and ``dQ = 0.125 dS K``,
``dK = 0.125 dS^T Q`` are exact before the bf16 output.  So ``dqkv`` must equal a float64 emulation bit for bit.  The
generator asserts these bounds, and that dS, dQ, dK and dV include rounding ties, which truncation and ties-away
rounding get wrong.  With dropout: ``dV = bf16(P o M s)^T dO``, ``dP' = M s o dP``, ``delta = rowsum(P o dP')`` with the
undropped P, ``dS = P o (dP' - delta)``.

Family F (full mantissa), fused kernels.  qkv is ``randn * 0.5`` rounded to bf16 with edge rows: all scores equal
(P = 1/128), one-hot rows, rows whose exp mostly underflows, scores near +100 and rows of only negative scores (a
constant key column times +-800).  u = 2^-24, t = scale q.k, a = scale sum_d |q_d k_d|, m the row max.  Per element:
* P~_k is exact up to a factor common to its row (the max and its rounding cancel in P~ / sum) and a relative
  ``rho_k = 2^-17 a_k + 4u |t_k - m| + 2^-21``: the fp32 score sum (64 terms), scale_log2e and the fma rounding, and
  ex2.approx.  The row sum adds 128 fp32 terms: ``sigma = sum_k P_k rho_k + 2^-17``.
* probs: a bf16 rounding of a value within ``P_k (rho_k + sigma + 4u)`` of P_k (P_k itself below 2^-120, flushed).
* out: a bf16 rounding of a value within ``sum_k P_k |v_k| (2^-8 + rho_k + 2^-17) + |o| (sigma + 4u)``: P~ is rounded
  to bf16 for the PV product while the row sum adds the unrounded values (a P~ below 2^-120 counts whole).
* every bf16 output gets ``2^-112`` more: fp32 products below 2^-120, up to 128 of them, may be flushed to zero.
* backward, with the bf16 P it is given: ``e_dP = 2^-17 sum_d |dO_d v_d|``, delta within
  ``2^-17 sum_k P_k |dP_k| + sum_k P_k e_dP_k``, dS within ``(2^-8 + 4u) |dS| + P (e_dP + e_delta)``; dQ (dK) within
  ``scale sum_k w_dS_k |K_k| + 2^-17 scale sum_k (|dS_k| + w_dS_k) |K_k|`` (of Q), dV within ``2^-17 sum_q P_q |dO_q|``.
The F tests print the worst error as a fraction of its window per output (``pytest -rP``; a bf16 output counts only
where it is not the nearest-even rounding of the reference), and the E tests the size of the ambiguity band.
Measured on one H100 80GB HBM3 at a 700 W power limit, worst over the cases and both dropout forms:
* family F: probs 0.017, out 0.82, dQ 0.86, dK 0.57, dV 0.029 (the multi-kernel path: out 0.95, dQ 0.95, dK 0.95,
  dV 0.89; a worst case near 1 is one bf16 rounding of a single dominant term at the bottom of its binade);
* family E: the band holds 4094 of 15.6 M ``out`` elements (0.026 %), 24 of which took the other neighbour, and
  14336 of 31.3 M ``probs`` elements (0.046 %), none of which did: consistent with ex2.approx returning exact powers
  of two on integer arguments, though not a proof of it, and no check relies on it.

Multi-kernel path.  qkv and dO are small integers; S in {64, 72, 128 (masked), 256, 512}, d_head in {32, 64}, batch
sizes on both sides of the batched GEMM's persistent switch (>= 2 x SMs tiles) and the model's key-padding mask of
-30000.  The reference rounds to bf16 where the path does: ``scores = RNE_bf16(fp32(alpha * QK^T))``, the mask added
in fp32 and rounded to bf16, probs, ``dprobs = RNE_bf16(dO V^T)`` and dscores.  The softmax kernels are within the
window of tests/test_gpu_norm_exact.py, so each probs (dscores) element is the nearest-even rounding of the float64
value or, inside that window of a rounding boundary, its neighbour: the reference carries that one-ulp deviation
through the GEMMs, plus ``2^-14 sum |terms|`` for their fp32 accumulation.  Padded keys get P = 0 exactly, and their
dK and dV rows are exactly zero.

The fused kernels' outputs are 16-byte-aligned slices of larger buffers filled with a NaN bit pattern: the guard
elements must keep their bits, and an element the kernel never writes stays NaN and fails.  The fused kernels have no
atomics: a second launch gives the same bits.  The attention bindings do not check the sizes of out, probs or dqkv."""
import math
import os
import re
import zlib
from collections import namedtuple
from functools import lru_cache

import numpy as np
import pytest
import torch

from baton_b200.data.dropout import DropoutRun, dropout_keep

BF16, F32, F64 = torch.bfloat16, torch.float32, torch.float64
U = 2.0 ** -24
BF16_U = 2.0 ** -8              # bf16 unit roundoff (8 significant bits)
S, DH = 128, 64
LN2_F32 = float(np.float32(math.log(2.0)))          # 0.693147182464599609375: fp32(ln 2) * fp32(log2 e) == 1.0
BWD_SCALE = 0.125
BAND = 2.0 ** -20                # relative: reciprocal and products (and a few ulp of ex2.approx) stay inside
ACC = 2.0 ** -17                 # fp32 chains of at most 128 terms (the fused kernels)
CHAIN = 2.0 ** -14               # fp32 chains of at most 512 terms (the multi-kernel path's GEMMs and row sums)
TINY = 2.0 ** -120               # below this a fp32 intermediate may be flushed
FLUSH = 256 * TINY               # absolute: up to 128 products below TINY (times s = 2) lost to flushing
EXACT_BOUND = 2 ** 24
P_DROP, DROP_SCALE = 0.5, 2.0
KEY, STREAM, SITE, EPOCH, STEP, STEPS = 0x5EED_0A77, (3 << 32) | 5, 1, 1, 2, 4
NAN_BITS = 0x7FC1
HEAD, TAIL = 8, 24               # guard elements before (16 bytes) and after every output

Case = namedtuple("Case", "id B H fams")
MCase = namedtuple("MCase", "id B H S dh mask")

# ------------------------------------------------------------------------------------------------ the case tables
FUSED = [
    Case("b1_h1", 1, 1, "EF"),
    Case("b1_h16", 1, 16, "E"),
    Case("b3_h2", 3, 2, "EF"),
    Case("b3_h12", 3, 12, "EF"),
    Case("b32_h12", 32, 12, "EF"),          # the BERT-base round at batch 32
    Case("b32_h16", 32, 16, "E"),
]
# batched-GEMM tiles: Q K^T and dO V^T are S x S (BN 128 when S > 64), the others S x d_head (BN 64); >= 2 x SMs tiles
# take the persistent kernel (264 on a 132-SM H100)
MULTI = [
    MCase("s64_d64", 2, 3, 64, 64, False),
    MCase("s64_d32_persistent", 24, 12, 64, 32, False),
    MCase("s72_d64", 3, 2, 72, 64, False),
    MCase("s128_d64_mask", 4, 12, 128, 64, True),
    MCase("s128_d64_mask_persistent", 24, 12, 128, 64, True),
    MCase("s256_d32", 2, 4, 256, 32, False),
    MCase("s512_d64_mask", 2, 2, 512, 64, True),
    MCase("s512_d32_persistent", 2, 9, 512, 32, False),
]
for _t in (FUSED, MULTI):
    assert len({c.id for c in _t}) == len(_t)


def _fcase(cid):
    return next(c for c in FUSED if c.id == cid)


def _gen(tag):
    return torch.Generator().manual_seed(zlib.crc32(tag.encode()))


# ------------------------------------------------------------------------------------------------ layouts
def _heads(qkv, B, H, which, dh=DH, s=S):
    """``[B*S, 3*H*dh]`` (which = 0, 1, 2: Q, K, V) or ``[B*S, H*dh]`` (which None) -> ``[B*H, S, dh]``."""
    x = qkv.reshape(B, s, -1, H, dh)
    x = x[:, :, which] if which is not None else x[:, :, 0]
    return x.permute(0, 2, 1, 3).reshape(B * H, s, dh)


def _pack(t, B, H):
    """``[B*H, S, dh]`` -> ``[B*S, H*dh]``."""
    nh, s, dh = t.shape
    return t.reshape(B, H, s, dh).permute(0, 2, 1, 3).reshape(B * s, H * dh)


def _pack_qkv(q, k, v, B, H):
    return torch.cat([_pack(q, B, H), _pack(k, B, H), _pack(v, B, H)], dim=1)


# ------------------------------------------------------------------------------------------------ bf16 rounding
def _frexp_grid(r):
    a = r.abs()
    _, e = torch.frexp(a)
    ulp = torch.ldexp(torch.ones_like(a), (e - 1).clamp_min(-126) - 7)
    return a / ulp, ulp


def _round_bf16(r, mode="rne"):
    q, ulp = _frexp_grid(r)
    m = {"rne": torch.round, "trunc": torch.floor, "away": lambda t: torch.floor(t + 0.5)}[mode](q)
    return torch.sign(r) * m * ulp


def _f32(t):
    return t.float().double()


def _min_bits(t):
    for b in range(0, 60):
        s = t * 2.0 ** b
        if torch.equal(s, s.round()):
            return b
    return 60


def _dyadic_ok(t, bits=None):
    """Every element of ``t`` (a sum of absolute terms) is below 2^24 units of 2^-bits."""
    b = _min_bits(t) if bits is None else bits
    return float(t.abs().max()) * 2.0 ** b < EXACT_BOUND


def _ties(r):
    rne = _round_bf16(r)
    return bool((_round_bf16(r, "trunc") != rne).any()) and bool((_round_bf16(r, "away") != rne).any())


# ------------------------------------------------------------------------------------------------ dropout mask
@lru_cache(maxsize=None)
def _keep_np(nh):
    return dropout_keep(KEY, STREAM, SITE, EPOCH * STEPS + STEP, nh * S * S, P_DROP).reshape(nh, S, S)


def _mask(nh, drop, dev="cpu"):
    """M s as float64 ``[nh, S, S]`` (ones without dropout)."""
    if not drop:
        return torch.ones(nh, S, S, dtype=F64, device=dev)
    return torch.from_numpy(_keep_np(nh)).to(dev).double() * DROP_SCALE


def _drop_args(dev):
    run = DropoutRun()
    run.begin(KEY, STREAM, STEPS, 3, 8)
    words = torch.tensor([EPOCH, STREAM & 0xFFFFFFFF, STREAM >> 32], dtype=torch.int64).to(torch.int32).to(dev)
    run.at(EPOCH, STEP, words)
    assert run.t == EPOCH * STEPS + STEP
    return run.kernel_args(SITE, P_DROP)


# ------------------------------------------------------------------------------------------------ data
def _sparse_int(shape, lo, hi, density, g):
    v = torch.randint(lo, hi + 1, shape, generator=g).double()
    return v * (torch.rand(shape, generator=g) < density).double()


def _sparse_pm1(shape, density, g):
    return torch.where(torch.rand(shape, generator=g) < 0.5, -1.0, 1.0).double() * \
        (torch.rand(shape, generator=g) < density).double()


def fwd_e_data(c):
    """Family E forward: q, k, v ``[B*H, S, 64]`` integers.  Key k is addressed by dims (k & 31) and 32 + (k >> 5);
    row r = 8 i + t of head number n puts A in {5, 6} on the address of key ``8 ((i + t + n) % 16) + t`` (its dominant
    key), noise lives on dims 36..63.  In heads n >= 1, rows with (r + n) % 32 == 7 are all zero (P = 1/128)."""
    g = _gen("fwdE/" + c.id)
    nh = c.B * c.H
    q = torch.zeros(nh, S, DH, dtype=F64)
    k = torch.zeros(nh, S, DH, dtype=F64)
    kk = torch.arange(S)
    k[:, kk, kk & 31] = 1.0
    k[:, kk, 32 + (kk >> 5)] = 1.0
    k[:, :, 36:] = _sparse_pm1((nh, S, 28), 0.2, g)
    q[:, :, 36:] = _sparse_pm1((nh, S, 28), 0.2, g)
    r = torch.arange(S)
    for n in range(nh):
        dom = 8 * (((r >> 3) + (r & 7) + n) % 16) + (r & 7)
        A = torch.randint(5, 7, (S,), generator=g).double()
        q[n, r, dom & 31] = A
        q[n, r, 32 + (dom >> 5)] = A
        if n >= 1:
            q[n, (r + n) % 32 == 7] = 0.0
    # a row whose noise spreads it beyond 16 binades, ties its maximum or takes its dominant key below 0.3 keeps its
    # address only
    x = q @ k.transpose(1, 2)
    P = torch.softmax(x * math.log(2.0), -1)
    top = P.max(-1).values
    bad = ((x.max(-1).values - x.min(-1).values) > 16) | (top < 0.3) | ((P == top[..., None]).sum(-1) > 1)
    q[:, :, 36:][bad] = 0.0
    v = _sparse_int((nh, S, DH), -2, 2, 0.8, g)
    return dict(q=q, k=k, v=v)


def bwd_e_data(c):
    """Family E backward: integer q, k, v, dO and a dyadic P (multiples of 1/128 up to 1/4, a third of them 0)."""
    g = _gen("bwdE/" + c.id)
    nh = c.B * c.H
    q, k, v = (_sparse_int((nh, S, DH), -2, 2, 0.5, g) for _ in range(3))
    do = _sparse_int((nh, S, DH), -2, 2, 0.5, g)
    P = _sparse_int((nh, S, S), 1, 32, 0.67, g) / 128.0
    return dict(q=q, k=k, v=v, do=do, P=P)


def f_data(c):
    """Family F: bf16(randn * 0.5) q, k, v and bf16(randn) dO; key column 63 is 1.0, and rows r % 16 = 1..5 are the
    edges: q = 0 (uniform), q = 16 k_r (one-hot), q = 64 k_r (most exp underflow), q_63 = +800 / -800 (scores near
    +100 / all near -100).  The backward's P is the float64 softmax rounded to bf16."""
    g = _gen("F/" + c.id)
    nh = c.B * c.H
    q, k, v, do = ((torch.randn(nh, S, DH, generator=g, dtype=F64) * (0.5 if i < 3 else 1.0)).to(BF16).double()
                   for i in range(4))
    k[:, :, 63] = 1.0
    r = torch.arange(S)
    q[:, r % 16 == 1] = 0.0
    q[:, r % 16 == 2] = 16.0 * k[:, r % 16 == 2]
    q[:, r % 16 == 3] = 64.0 * k[:, r % 16 == 3]
    q[:, r % 16 == 4, 63] = 800.0
    q[:, r % 16 == 5, 63] = -800.0
    t = 0.125 * q @ k.transpose(1, 2)
    P = _round_bf16(torch.softmax(t, -1))
    return dict(q=q, k=k, v=v, do=do, P=P)


def multi_data(c):
    """Multi-kernel path: integer q, k, v, dO in [-2, 2] ``[B*H, S, dh]`` and, with a mask, per batch element a count
    of attended keys (at least 1) -- the model's ``(1 - attention_mask) * -30000``."""
    g = _gen("M/" + c.id)
    nh = c.B * c.H
    q, k, v, do = (_sparse_int((nh, c.S, c.dh), -2, 2, 0.7, g) for _ in range(4))
    mask = None
    if c.mask:
        n_att = torch.randint(1, c.S + 1, (c.B,), generator=g)
        n_att[0] = c.S
        n_att[-1] = min(int(n_att[-1]), 3)
        am = (torch.arange(c.S)[None, :] < n_att[:, None]).float()
        mask = (1.0 - am) * -30000.0
    return dict(q=q, k=k, v=v, do=do, mask=mask)


# ------------------------------------------------------------------------------------------------ references
def ref_fwd_e(d, M):
    """Exact float64 P, out, and P~ / row sums (M = mask times s, or ones)."""
    x = d["q"] @ d["k"].transpose(1, 2)
    m = x.max(-1, keepdim=True).values
    Pt = torch.exp2(x - m)
    sm = Pt.sum(-1, keepdim=True)
    return dict(x=x, Pt=Pt, sum=sm, P=Pt / sm, out=((Pt * M) @ d["v"]) / sm)


def emu_bwd_e(d, M, mode="rne", delta_skip=None, delta_dropped=False):
    """Bit-exact float64 emulation of the fused backward on family E data: ``dS = round(P (dP' - delta))``, the rest
    exact before the bf16 outputs.  The keyword arguments build the mistakes the sensitivity test rejects."""
    P = d["P"]
    dP = M * (d["do"] @ d["v"].transpose(1, 2))
    Pd = P * M if delta_dropped else P
    t = Pd * dP
    if delta_skip is not None:
        t = t.clone()
        t[:, :, delta_skip] = 0.0
    delta = t.sum(-1, keepdim=True)
    dS = _round_bf16(P * (dP - delta), mode)
    dq = BWD_SCALE * dS @ d["k"]
    dk = BWD_SCALE * dS.transpose(1, 2) @ d["q"]
    dv = (P * M).transpose(1, 2) @ d["do"]
    return dict(dP=dP, delta=delta, dS_exact=P * (dP - delta), dS=dS, dq=dq, dk=dk, dv=dv)


def ref_fwd_f(d, M, scale=0.125):
    q, k, v = d["q"], d["k"], d["v"]
    t = scale * q @ k.transpose(1, 2)
    a = scale * q.abs() @ k.abs().transpose(1, 2)
    m = t.max(-1, keepdim=True).values
    e = torch.exp(t - m)
    P = e / e.sum(-1, keepdim=True)
    rho = ACC * a + 4 * U * (t - m).abs() + 2.0 ** -21
    sigma = (P * rho).sum(-1, keepdim=True) + ACC
    PM = P * M
    out = PM @ v
    rel = torch.where(e < TINY, torch.ones_like(e), BF16_U + rho + ACC)
    w_out = (PM * rel) @ v.abs() + out.abs() * (sigma + 4 * U) + FLUSH
    w_p = torch.where(P < TINY, P, P * (rho + sigma + 4 * U))
    return dict(P=P, out=out, w_p=w_p, w_out=w_out)


def ref_bwd_f(d, M, scale=0.125):
    q, k, v, do, P = d["q"], d["k"], d["v"], d["do"], d["P"]
    dP = M * (do @ v.transpose(1, 2))
    e_dP = M * ACC * (do.abs() @ v.abs().transpose(1, 2))
    delta = (P * dP).sum(-1, keepdim=True)
    e_d = ACC * (P * dP.abs()).sum(-1, keepdim=True) + (P * e_dP).sum(-1, keepdim=True)
    dS = P * (dP - delta)
    w_dS = (BF16_U + 4 * U) * dS.abs() + 1.01 * P * (e_dP + e_d) + TINY
    dq = scale * dS @ k
    w_dq = scale * (w_dS @ k.abs() + ACC * (dS.abs() + w_dS) @ k.abs()) + U * dq.abs() + FLUSH
    dk = scale * dS.transpose(1, 2) @ q
    w_dk = scale * (w_dS.transpose(1, 2) @ q.abs() + ACC * (dS.abs() + w_dS).transpose(1, 2) @ q.abs()) + U * dk.abs() \
        + FLUSH
    PM = P * M
    dv = PM.transpose(1, 2) @ do
    w_dv = ACC * PM.transpose(1, 2) @ do.abs() + FLUSH
    return dict(dq=dq, dk=dk, dv=dv, w_dq=w_dq, w_dk=w_dk, w_dv=w_dv)


def _dev(ref, w):
    """The bf16 values within ``w`` of ``ref``: the nearest-even one and its largest distance to the others."""
    r0 = _round_bf16(ref)
    return r0, torch.maximum((_round_bf16(ref + w) - r0).abs(), (_round_bf16(ref - w) - r0).abs())


def ref_multi(c, d):
    """The multi-kernel path in float64 with its bf16 roundings: -> the references and windows of out, dq, dk, dv."""
    q, k, v, do = d["q"], d["k"], d["v"], d["do"]
    alpha = _f32(torch.tensor(1.0 / math.sqrt(c.dh), dtype=F64))
    sc = _round_bf16(_f32(alpha * (q @ k.transpose(1, 2))))
    pad = None
    if d["mask"] is not None:
        mb = d["mask"].to(BF16).double().to(q.device)                      # -30000 -> -29952
        mb = mb.repeat_interleave(c.H, 0)[:, None, :]
        sc = _round_bf16(_f32(sc + mb))
        pad = (mb < 0).expand_as(sc)
    m = sc.max(-1, keepdim=True).values
    e = torch.exp(sc - m)
    p = e / e.sum(-1, keepdim=True)
    a = sc.abs() + (sc - m).abs()
    w_p = p * U * (16 + c.S + 2 * a + (p * (8 + 2 * a)).sum(-1, keepdim=True))
    w_p = torch.where(p < TINY, p, w_p)
    P0, dvP = _dev(p, w_p)
    out = P0 @ v
    w_out = dvP @ v.abs() + CHAIN * P0 @ v.abs()
    dv = P0.transpose(1, 2) @ do
    w_dv = dvP.transpose(1, 2) @ do.abs() + CHAIN * P0.transpose(1, 2) @ do.abs()
    g = _round_bf16(do @ v.transpose(1, 2))
    s = (P0 * g).sum(-1, keepdim=True)
    dS = P0 * (g - s)
    spread = (dvP * g.abs()).sum(-1, keepdim=True)
    W = dvP * ((g - s).abs() + spread) + (P0 + dvP) * spread + 1.01 * P0 * CHAIN * (P0 * g).abs().sum(-1, keepdim=True) \
        + 4 * U * dS.abs()
    S0, dvS = _dev(dS, W)
    dq = alpha * S0 @ k
    w_dq = alpha * (dvS @ k.abs() + CHAIN * (S0.abs() + dvS) @ k.abs()) + U * dq.abs()
    dk = alpha * S0.transpose(1, 2) @ q
    w_dk = alpha * (dvS.transpose(1, 2) @ q.abs() + CHAIN * (S0.abs() + dvS).transpose(1, 2) @ q.abs()) + U * dk.abs()
    return dict(out=out, w_out=w_out, dq=dq, w_dq=w_dq, dk=dk, w_dk=w_dk, dv=dv, w_dv=w_dv, P0=P0, pad=pad)


# ------------------------------------------------------------------------------------------------ checks
def _mismatch(tag, got, ref, bad):
    idx = bad.nonzero()[:5].tolist()
    return "{}: {} of {} elements differ, first at {}: got {} want {}".format(
        tag, int(bad.sum()), bad.numel(), idx, [float(got[tuple(i)]) for i in idx], [float(ref[tuple(i)]) for i in idx])


def check_bf16(tag, got, ref, w=None):
    """A bf16 ``got`` is the correct rounding of some value within ``w`` of ``ref`` (w None: ``ref`` rounded to
    nearest-even).  Returns the worst distance from a value that rounds to ``got``, as a fraction of ``w``."""
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


def check_band(tag, got, ref):
    """Nearest-even bf16 of ``ref``, or either neighbour inside the ``BAND`` of a rounding boundary.  -> (elements in
    the band, band elements that took the other neighbour)."""
    w = BAND * ref.abs()
    check_bf16(tag, got, ref, w)
    band = _round_bf16(ref - w) != _round_bf16(ref + w)
    return int(band.sum()), int((band & (got.double() != _round_bf16(ref))).sum())


def check_fwd_e(tag, c, out, probs, ref):
    """-> {output: (band, other neighbour)}; out ``[B*S, H*64]``, probs ``[B*H*S, S]``."""
    return {"out": check_band(tag + " out", out, _pack(ref["out"], c.B, c.H)),
            "probs": check_band(tag + " probs", probs, ref["P"].reshape(-1, S))}


def check_bwd_e(tag, c, dqkv, emu):
    check_bf16(tag + " dqkv", dqkv, _pack_qkv(emu["dq"], emu["dk"], emu["dv"], c.B, c.H))


def check_fwd_f(tag, c, out, probs, ref):
    return {"probs": check_bf16(tag + " probs", probs, ref["P"].reshape(-1, S), ref["w_p"].reshape(-1, S)),
            "out": check_bf16(tag + " out", out, _pack(ref["out"], c.B, c.H), _pack(ref["w_out"], c.B, c.H))}


def check_grads(tag, B, H, dqkv, ref):
    D = dqkv.shape[1] // 3
    r = {}
    for i, n in enumerate(("dq", "dk", "dv")):
        r[n] = check_bf16(tag + " " + n, dqkv[:, i * D:(i + 1) * D], _pack(ref[n], B, H), _pack(ref["w_" + n], B, H))
    return r


# ------------------------------------------------------------------------------------------------ CPU: the generator
def test_fp32_ln2_scale_makes_scale_log2e_one():
    s = np.float32(LN2_F32)
    assert LN2_F32 == 0.693147182464599609375
    assert np.float32(s * np.float32(1.4426950408889634)) == np.float32(1.0)


def _fwd_e_asserts(c, d, ref):
    x, Pt, P, v = ref["x"], ref["Pt"], ref["P"], d["v"]
    assert torch.equal(x, x.round()), c.id
    E = float((x.max(-1).values - x.min(-1).values).max())
    assert E <= 16, (c.id, E)
    assert float((Pt @ v.abs()).max()) * 2.0 ** 16 < EXACT_BOUND, c.id
    top = P.max(-1)
    unique = (P == top.values[..., None]).sum(-1) == 1
    dom = top.indices[(top.values >= 0.25) & unique]
    assert set(dom.unique().tolist()) == set(range(S)), c.id
    r = torch.arange(S)[None, :, None].expand_as(P)
    key = torch.arange(S)[None, None, :].expand_as(P)
    carry = (P >= 0.25) & (v.abs().sum(-1) > 0)[:, None, :]
    pairs = set(zip((((key & 63) >> 3)[carry]).tolist(), ((r & 7)[carry]).tolist()))
    assert pairs == {(ch, t) for ch in range(8) for t in range(8)}, c.id


def _bwd_e_asserts(c, d, M, emu):
    bits = _min_bits(emu["dS"])
    assert bits <= 14, c.id
    assert _dyadic_ok((d["P"] * emu["dP"].abs()).sum(-1), 7), c.id                 # delta's fma chain
    assert torch.equal(emu["dS_exact"], _f32(emu["dS_exact"])), c.id               # P (dP - delta) exact in fp32
    assert _dyadic_ok(emu["dS"].abs() @ d["k"].abs(), bits), c.id
    assert _dyadic_ok(emu["dS"].abs().transpose(1, 2) @ d["q"].abs(), bits), c.id
    assert _dyadic_ok((d["P"] * M).transpose(1, 2) @ d["do"].abs(), 7), c.id
    for n in ("dS_exact", "dq", "dk", "dv"):
        assert _ties(emu[n]), (c.id, n)


def test_generator_bounds_ties_and_coverage():
    """Family E data of every fused case, with and without dropout: the exactness bounds, the dominant keys and
    swizzle coverage of the forward, the rounding ties of the backward; and the F data's edge rows."""
    for c in FUSED:
        nh = c.B * c.H
        for drop in (False, True):
            M = _mask(nh, drop)
            d = fwd_e_data(c)
            _fwd_e_asserts(c, d, ref_fwd_e(d, M))
            db = bwd_e_data(c)
            _bwd_e_asserts(c, db, M, emu_bwd_e(db, M))
        if "F" in c.fams:
            d = f_data(c)
            ref = ref_fwd_f(d, _mask(nh, False))
            r = torch.arange(S)
            assert bool((ref["P"][:, r % 16 == 1] == 1.0 / S).all())
            assert bool((ref["P"][:, r % 16 == 2].max(-1).values > 0.99).all())
            assert float((ref["P"][:, r % 16 == 3] < TINY).double().mean()) > 0.5
            t = 0.125 * d["q"] @ d["k"].transpose(1, 2)
            assert bool((t[:, r % 16 == 4].min(-1).values > 90).all())
            assert bool((t[:, r % 16 == 5].max(-1).values < -90).all())


def test_multi_kernel_table_covers_both_sides_of_the_persistent_switch():
    kernels = set().union(*(_multi_kernels(c, 132) for c in MULTI))
    assert {"persistent<128,3>", "persistent<64,5>", "fixed<128,6>", "fixed<64,8>"} <= kernels, kernels
    assert {"softmax_fwd_vec<{},{}>".format(*lv) for lv in [(8, 1), (16, 1), (32, 1), (32, 2)]} <= kernels, kernels
    assert {c.S for c in MULTI} == {64, 72, 128, 256, 512} and {c.dh for c in MULTI} == {32, 64}
    assert all(c.mask for c in MULTI if c.S == 128)
    for c in MULTI:                    # every softmax window stays below a bf16 ulp, and padded keys get exactly 0
        d = multi_data(c)
        ref = ref_multi(c, d)
        if c.mask:
            assert bool((ref["P0"][ref["pad"]] == 0).all()) and bool(ref["pad"].any()), c.id


def _multi_kernels(c, sms):
    def pick(bn, tiles):
        if tiles >= 2 * sms:
            return "persistent<128,3>" if bn == 128 else "persistent<64,5>"
        return "fixed<128,6>" if bn == 128 else "fixed<64,8>"
    nh = c.B * c.H
    bn = 128 if c.S > 64 else 64
    mt = (c.S + 127) // 128
    nvec = c.S // 8
    lv = (8, 1) if nvec <= 8 else (16, 1) if nvec <= 16 else (32, 1) if nvec <= 32 else (32, 2) if nvec <= 64 else None
    return {pick(bn, ((c.S + bn - 1) // bn) * mt * nh), pick(64, mt * nh), "softmax_fwd_vec<{},{}>".format(*lv),
            "softmax_bwd_vec<{},{}>".format(*lv)}


# ------------------------------------------------------------------------------------------------ CPU: sensitivity
def test_checks_reject_plausible_mistakes():
    """On the CPU, in float64: each mistake below makes a 'kernel output' that the checks of this module reject, on
    the case data they run on the GPU."""
    c = _fcase("b3_h2")
    nh = c.B * c.H
    one, Md = _mask(nh, False), _mask(nh, True)
    for M, drop in ((one, False), (Md, True)):
        d = fwd_e_data(c)
        ref = ref_fwd_e(d, M)
        good = (_round_bf16(_pack(ref["out"], c.B, c.H)), _round_bf16(ref["P"].reshape(-1, S)))
        check_fwd_e("exact", c, *good, ref)
        O = (ref["Pt"] * M) @ d["v"]
        # the row sum skips key 77, P~ keeps it
        sm = ref["sum"] - ref["Pt"][:, :, 77:78]
        bad = (_round_bf16(_pack(O / sm, c.B, c.H)), _round_bf16((ref["Pt"] / sm).reshape(-1, S)))
        with pytest.raises(AssertionError):
            check_fwd_e("row sum without a key", c, *bad, ref)
        # key 77 dropped from P~ in the rows of one swizzle phase (r & 7 == 5); the row sum keeps it
        Pt = ref["Pt"].clone()
        Pt[:, 5::8, 77] = 0.0
        with pytest.raises(AssertionError):
            check_fwd_e("P~ without a key", c, _round_bf16(_pack((Pt * M) @ d["v"] / ref["sum"], c.B, c.H)), good[1], ref)
        # two heads swapped in out
        o = ref["out"].clone()
        o[[0, 1]] = o[[1, 0]]
        with pytest.raises(AssertionError):
            check_fwd_e("heads swapped", c, _round_bf16(_pack(o, c.B, c.H)), good[1], ref)
        if drop:   # saved probs that include the dropout scale
            with pytest.raises(AssertionError):
                check_fwd_e("probs times M s", c, good[0], _round_bf16((ref["P"] * Md).reshape(-1, S)), ref)
        db = bwd_e_data(c)
        emu = emu_bwd_e(db, M)
        check_bwd_e("exact", c, _pack_qkv(*(_round_bf16(emu[n]) for n in ("dq", "dk", "dv")), c.B, c.H), emu)
        bads = {"truncated dS": emu_bwd_e(db, M, mode="trunc"), "ties-away dS": emu_bwd_e(db, M, mode="away"),
                "delta without a key": emu_bwd_e(db, M, delta_skip=77)}
        if drop:
            bads["delta from the dropped P"] = emu_bwd_e(db, M, delta_dropped=True)
        for what, e in bads.items():
            got = _pack_qkv(*(_round_bf16(e[n]) for n in ("dq", "dk", "dv")), c.B, c.H)
            with pytest.raises(AssertionError):
                check_bwd_e(what, c, got, emu)
        # family F: the same mistakes against the bounded windows
        d = f_data(c)
        ref = ref_fwd_f(d, M)
        check_fwd_f("F", c, _round_bf16(_pack(ref["out"], c.B, c.H)), _round_bf16(ref["P"].reshape(-1, S)), ref)
        o = ref["out"].clone()
        o[[0, 1]] = o[[1, 0]]
        with pytest.raises(AssertionError):
            check_fwd_f("F heads swapped", c, _round_bf16(_pack(o, c.B, c.H)), _round_bf16(ref["P"].reshape(-1, S)), ref)
        rb = ref_bwd_f(d, M)
        got = _pack_qkv(*(_round_bf16(rb[n]) for n in ("dq", "dk", "dv")), c.B, c.H)
        check_grads("F", c.B, c.H, got, rb)
        dP = M * (d["do"] @ d["v"].transpose(1, 2))
        t = d["P"] * dP
        t[:, :, 77] = 0.0
        dS = d["P"] * (dP - t.sum(-1, keepdim=True))
        bad = _pack_qkv(_round_bf16(BWD_SCALE * dS @ d["k"]), _round_bf16(rb["dk"]), _round_bf16(rb["dv"]), c.B, c.H)
        with pytest.raises(AssertionError):
            check_grads("F delta without a key", c.B, c.H, bad, rb)
    # the multi-kernel path: a mask ignored, the head strides of dqkv swapped
    c = next(m for m in MULTI if m.id == "s128_d64_mask")
    d = multi_data(c)
    ref = ref_multi(c, d)
    got = _pack_qkv(*(_round_bf16(ref[n]) for n in ("dq", "dk", "dv")), c.B, c.H)
    check_grads("M", c.B, c.H, got, ref)
    check_bf16("M out", _round_bf16(_pack(ref["out"], c.B, c.H)), _pack(ref["out"], c.B, c.H), _pack(ref["w_out"], c.B, c.H))
    nomask = ref_multi(c, dict(d, mask=None))
    with pytest.raises(AssertionError):
        check_bf16("M out without mask", _round_bf16(_pack(nomask["out"], c.B, c.H)), _pack(ref["out"], c.B, c.H),
                   _pack(ref["w_out"], c.B, c.H))
    dk = ref["dk"].clone()
    dk[[0, 1]] = dk[[1, 0]]
    with pytest.raises(AssertionError):
        check_grads("M dk heads swapped", c.B, c.H, _pack_qkv(*(_round_bf16(t) for t in (ref["dq"], dk, ref["dv"])),
                                                              c.B, c.H), ref)


# ------------------------------------------------------------------------------------------------ GPU
@pytest.fixture(scope="module")
def C_():
    from baton_b200.ops import load
    return load()


def _guarded(shape, dev):
    """A ``shape`` bf16 view at a 16-byte offset of a buffer filled with the NaN sentinel -> (view, check)."""
    n = math.prod(shape)
    buf = torch.full((HEAD + n + TAIL,), NAN_BITS, dtype=torch.int16, device=dev)
    view = buf[HEAD: HEAD + n].view(BF16).view(shape)
    assert view.data_ptr() % 16 == 0

    def check(tag):
        guard = torch.cat([buf[:HEAD], buf[HEAD + n:]])
        assert bool((guard == NAN_BITS).all()), tag + ": guard elements overwritten"
    return view, check


def _bf(t, dev):
    return t.to(dev).to(BF16)


def _run_fused(C_, c, d, drop, scale, fwd, dev):
    """One fused launch into guarded buffers -> (outputs, guard checks)."""
    B, H = c.B, c.H
    D = H * DH
    qkv = _bf(_pack_qkv(d["q"], d["k"], d["v"], B, H), dev)
    da = _drop_args(dev) if drop else None
    if fwd:
        out, co = _guarded((B * S, D), dev)
        probs, cp = _guarded((B * H * S, S), dev)
        ok = (C_.attention_drop_fwd(qkv, out, probs, B, S, H, DH, scale, *da) if drop else
              C_.attention_fwd(qkv, out, probs, B, S, H, DH, scale))
        assert ok
        return dict(out=out, probs=probs), [co, cp]
    dqkv, cd = _guarded((B * S, 3 * D), dev)
    dout = _bf(_pack(d["do"], B, H), dev)
    P = _bf(d["P"].reshape(-1, S), dev)
    ok = (C_.attention_drop_bwd(qkv, dout, P, dqkv, B, S, H, DH, scale, *da) if drop else
          C_.attention_bwd(qkv, dout, P, dqkv, B, S, H, DH, scale))
    assert ok
    return dict(dqkv=dqkv), [cd]


def _launch_twice(C_, c, d, drop, scale, fwd, dev):
    a, checks = _run_fused(C_, c, d, drop, scale, fwd, dev)
    b, checks2 = _run_fused(C_, c, d, drop, scale, fwd, dev)
    torch.cuda.synchronize()
    for n in a:
        assert torch.equal(a[n].view(torch.int16), b[n].view(torch.int16)), "{} {}: two launches differ".format(c.id, n)
    for chk in checks + checks2:
        chk(c.id)
    return {n: t.double() for n, t in a.items()}


E_PARAMS = [pytest.param(c, drop, id="{}-{}".format(c.id, "drop" if drop else "nodrop"))
            for c in FUSED for drop in (False, True)]
F_PARAMS = [p for p in E_PARAMS if "F" in p.values[0].fams]


@pytest.mark.gpu
@pytest.mark.parametrize("case,drop", E_PARAMS)
def test_fused_exact_dyadic_operands(C_, case, drop):
    dev = torch.device("cuda:0")
    nh = case.B * case.H
    M = _mask(nh, drop, dev)
    d = {n: t.to(dev) for n, t in fwd_e_data(case).items()}
    got = _launch_twice(C_, case, d, drop, LN2_F32, True, dev)
    band = check_fwd_e(case.id, case, got["out"], got["probs"], ref_fwd_e(d, M))
    n_out, n_p = got["out"].numel(), got["probs"].numel()
    assert band["out"][0] <= n_out // 64 and band["probs"][0] <= n_p // 64, band
    print("{}: band (elements, other neighbour taken): out {} of {}, probs {} of {}".format(
        case.id, band["out"], n_out, band["probs"], n_p))
    db = {n: t.to(dev) for n, t in bwd_e_data(case).items()}
    got = _launch_twice(C_, case, db, drop, BWD_SCALE, False, dev)
    check_bwd_e(case.id, case, got["dqkv"], emu_bwd_e(db, M))


@pytest.mark.gpu
@pytest.mark.parametrize("case,drop", F_PARAMS)
def test_fused_full_mantissa_operands(C_, case, drop):
    dev = torch.device("cuda:0")
    M = _mask(case.B * case.H, drop, dev)
    d = {n: t.to(dev) for n, t in f_data(case).items()}
    got = _launch_twice(C_, case, d, drop, 0.125, True, dev)
    r = check_fwd_f(case.id, case, got["out"], got["probs"], ref_fwd_f(d, M))
    got = _launch_twice(C_, case, d, drop, 0.125, False, dev)
    r.update(check_grads(case.id, case.B, case.H, got["dqkv"], ref_bwd_f(d, M)))
    print("{} (F): worst error / window: {}".format(case.id, ", ".join("{} {:.3g}".format(k, v) for k, v in r.items())))


def _run_multi(c, d, dev):
    from baton_b200.ops import nn as bnn
    qkv = _bf(_pack_qkv(d["q"], d["k"], d["v"], c.B, c.H), dev).requires_grad_(True)
    mask = d["mask"].to(dev) if d["mask"] is not None else None
    out = bnn.attention(qkv, c.B, c.S, c.H, c.dh, mask_bias=mask)
    out.backward(_bf(_pack(d["do"], c.B, c.H), dev))
    return out.detach(), qkv.grad


@pytest.mark.gpu
@pytest.mark.parametrize("case", MULTI, ids=[c.id for c in MULTI])
def test_multi_kernel_path(case):
    dev = torch.device("cuda:0")
    d = {n: (t.to(dev) if t is not None else None) for n, t in multi_data(case).items()}
    out, dqkv = _run_multi(case, d, dev)
    torch.cuda.synchronize()
    ref = ref_multi(case, d)
    r = {"out": check_bf16(case.id + " out", out, _pack(ref["out"], case.B, case.H), _pack(ref["w_out"], case.B, case.H))}
    r.update(check_grads(case.id, case.B, case.H, dqkv, ref))
    if case.mask:
        D = case.H * case.dh
        padded = (d["mask"] < 0).reshape(-1)
        assert bool((dqkv[padded, D:] == 0).all()), case.id + ": dK / dV rows of padded keys"
    print("{}: worst error / window: {}".format(case.id, ", ".join("{} {:.3g}".format(k, v) for k, v in r.items())))


_KERNEL = re.compile(r"b200::(attention_fwd_s128|attention_bwd_s128|gemm_bf16_fixed|gemm_bf16_persistent|softmax_fwd_vec|"
                     r"softmax_bwd_vec)_kernel<([^>]*)>")


def _kernel_key(name):
    m = _KERNEL.search(name)
    if m is None:
        return None
    args = [{"true": "1", "false": "0"}.get(a, a) for a in (re.sub(r"^\(\w+\)", "", x.strip()) for x in m.group(2).split(","))]
    base = m.group(1)
    if base.startswith("attention"):
        return "{}<{}>".format(base, args[0])
    if base.startswith("gemm_bf16_"):
        return "{}<{},{}>".format(base[len("gemm_bf16_"):], args[0], args[1])
    return "{}<{},{}>".format(base, args[0], args[1])


def test_kernel_key_parses_demangled_names():
    assert _kernel_key("void b200::attention_fwd_s128_kernel<true>(CUtensorMap_st, CUtensorMap_st, ...)") == \
        "attention_fwd_s128<1>"
    assert _kernel_key("void b200::attention_bwd_s128_kernel<(bool)0>(CUtensorMap_st, ...)") == "attention_bwd_s128<0>"
    assert _kernel_key("void b200::gemm_bf16_fixed_kernel<128, 6, 0, false, false, false, false, false>(...)") == \
        "fixed<128,6>"
    assert _kernel_key("void b200::gemm_bf16_persistent_kernel<64, 5>(CUtensorMap_st, ...)") == "persistent<64,5>"
    assert _kernel_key("void b200::softmax_bwd_vec_kernel<32, 2>(__nv_bfloat16 const*, ...)") == "softmax_bwd_vec<32,2>"


def _attention_globals():
    src = open(os.path.join(os.path.dirname(__file__), "..", "baton_b200", "csrc", "attention.cu")).read()
    return set(re.findall(r"__global__ void __launch_bounds__\([^)]*\)\s+(\w+)_kernel\(", src))


def _profiled(fn):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return {_kernel_key(e.name) for e in prof.events()} - {None}


@pytest.mark.gpu
def test_case_table_reaches_every_kernel(C_):
    """Under torch.profiler: every ``__global__`` of attention.cu runs with both DROP values, and each multi-kernel
    case runs the batched GEMM variants and softmax row kernels it names (and no fused kernel)."""
    dev = torch.device("cuda:0")
    c = _fcase("b3_h2")

    def fused():
        for drop in (False, True):
            _run_fused(C_, c, {n: t.to(dev) for n, t in fwd_e_data(c).items()}, drop, LN2_F32, True, dev)
            _run_fused(C_, c, {n: t.to(dev) for n, t in bwd_e_data(c).items()}, drop, BWD_SCALE, False, dev)
    globals_ = _attention_globals()
    assert globals_ == {"attention_fwd_s128", "attention_bwd_s128"}, globals_
    seen = _profiled(fused)
    want = {"{}<{}>".format(g, b) for g in globals_ for b in (0, 1)}
    assert want <= seen, sorted(want - seen)
    sms = torch.cuda.get_device_properties(dev).multi_processor_count
    for m in MULTI:
        d = {n: (t.to(dev) if t is not None else None) for n, t in multi_data(m).items()}
        seen = _profiled(lambda: _run_multi(m, d, dev))
        want = _multi_kernels(m, sms)
        assert want <= seen, (m.id, sorted(want - seen))
        assert not any(k.startswith("attention") for k in seen), (m.id, seen)
