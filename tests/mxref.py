"""Independent float64 reference of the project's MXFP8 format: the quantisers of ``csrc/quant.cu`` and the
block-scaled GEMM of ``csrc/gemm_fp8.cu``, written from the format's definition in plain torch (no project import),
so that a kernel and this module cannot agree on a mistake.

The format, as ``csrc/mx.cuh`` defines it:

* One shared exponent ``e`` per 32 consecutive elements along the GEMM's reduction axis.  ``amax`` is the block's
  largest magnitude; NaN is skipped, as ``fmaxf`` does.  ``e = floor(log2 amax) - 8``, plus one when amax's mantissa
  is strictly above 1.75, so that ``amax * 2^-e`` never exceeds 448 and the block maximum never saturates.  This
  bump rule is the project's own: the OCP MX specification takes ``floor(log2 amax) - 8`` and lets the block maximum
  saturate.  ``e`` is clamped to [-127, 127].  A block whose amax is zero (or all NaN) gets ``e = -127``.  The kernel
  reads the exponent field of amax's bits, so ``+-inf`` counts as ``2^128`` and gives ``e = 120``.
* The scale byte is ``e + 127`` (UE8M0).
* Each element is ``x * 2^-e`` rounded to nearest-even into e4m3 and saturated to +-448: ``+-inf`` becomes +-448 and
  NaN stays NaN (byte 0x7F).
* The extension is built with ``--use_fast_math``: fp32 denormals are flushed to zero, so a bf16 input below 2^-126
  counts as (a signed) zero, both in amax and as an element.
* Scales are stored in 512-byte atoms, one per 128 rows x 128 reduction elements:
  ``atom(row // 128, k // 128)[(row % 32) * 16 + ((row % 128) // 32) * 4 + (k % 128) // 32]``.  Padding rows and
  padding blocks of a partial atom hold byte 0.
* The GEMM decodes a scale byte ``b`` as ``2^(b - 127)``, except byte 0, which it decodes as 0.0 (the bit pattern
  ``b << 23``), not as 2^-127.  Its fp32 scale product ``sa * sb`` also flushes below 2^-126; callers that compare
  against :func:`gemm` keep their operands in ranges where that cannot happen.
"""
import math

import torch

E4M3_MAX = 448.0
SF_ATOM = 512
FP32_MIN_NORMAL = 2.0 ** -126


def _ceil(a: int, b: int) -> int:
    return (a + b - 1) // b


def flush_denormals(x: torch.Tensor) -> torch.Tensor:
    """float64 copy of ``x`` with |values| below 2^-126 replaced by a zero of the same sign (NaN and inf kept)."""
    x = x.to(torch.float64)
    return torch.where(x.abs() < FP32_MIN_NORMAL, x * 0.0, x)


def block_exponent(amax: torch.Tensor) -> torch.Tensor:
    """Shared exponent (int64) of blocks whose largest magnitude is ``amax`` (float64, >= 0, NaN already skipped)."""
    finite = torch.where(torch.isfinite(amax), amax, torch.ones_like(amax))
    m, ex = torch.frexp(finite)                       # finite = m * 2^ex, m in [0.5, 1): floor(log2) = ex - 1
    e = ex.to(torch.int64) - 1 - 8 + (2.0 * m > 1.75).to(torch.int64)
    e = torch.where(torch.isinf(amax), torch.full_like(e, 128 - 8), e)
    e = e.clamp(-127, 127)
    return torch.where(amax > 0, e, torch.full_like(e, -127))


def encode_e4m3(t: torch.Tensor) -> torch.Tensor:
    """float64 -> e4m3 bytes (uint8): round to nearest-even, saturate to +-448, NaN -> 0x7F.  torch's
    ``float8_e4m3fn`` cast rounds to nearest-even but returns NaN above 464 instead of saturating, so clamp first."""
    q = t.clamp(-E4M3_MAX, E4M3_MAX).to(torch.float32).to(torch.float8_e4m3fn).view(torch.uint8)
    return torch.where(torch.isnan(t), torch.full_like(q, 0x7F), q)


def decode_e4m3(q: torch.Tensor) -> torch.Tensor:
    return q.view(torch.float8_e4m3fn).to(torch.float32).to(torch.float64)


def _quant_last(x: torch.Tensor):
    """Blocks of 32 along the last axis of ``x`` ([R, C], C % 32 == 0): (q bytes [R, C], exponents [R, C // 32])."""
    R, C = x.shape
    blocks = x.reshape(R, C // 32, 32)
    a = blocks.abs()
    amax = torch.where(torch.isnan(a), torch.zeros_like(a), a).amax(-1)
    e = block_exponent(amax)
    q = encode_e4m3(blocks * torch.exp2(-e.to(torch.float64)).unsqueeze(-1))
    return q.reshape(R, C), e


def atoms(exps: torch.Tensor) -> torch.Tensor:
    """Exponents [Rpad, Kb] (Rpad % 128 == 0, Kb % 4 == 0) -> scale bytes in the 512-byte atom layout."""
    Rpad, Kb = exps.shape
    b = (exps + 127).to(torch.uint8).reshape(Rpad // 128, 4, 32, Kb // 4, 4)   # [row tile, row%128//32, row%32, k tile, kb%4]
    return b.permute(0, 3, 2, 1, 4).reshape(-1).contiguous()


def scales_of(sf: torch.Tensor, rows: int, K: int) -> torch.Tensor:
    """Inverse of :func:`atoms`: per-element float64 scales [rows, K] as the GEMM decodes them (byte 0 -> 0.0)."""
    rt, kt = _ceil(rows, 128), _ceil(K, 128)
    b = sf[: rt * kt * SF_ATOM].reshape(rt, kt, 32, 4, 4).permute(0, 3, 2, 1, 4).reshape(rt * 128, kt * 4)
    b = b[:rows, : _ceil(K, 32)].to(torch.int64)
    s = torch.where(b == 0, torch.zeros((), dtype=torch.float64, device=sf.device), torch.exp2((b - 127).to(torch.float64)))
    return s.repeat_interleave(32, dim=1)[:, :K]


def _quant(x2: torch.Tensor, keep_rows: int, keep_cols: int):
    """Quantise rows of ``x2`` ([rows, k], blocks along k): the q buffer [keep_rows, keep_cols] and the scale atoms,
    padding included."""
    rows, k = x2.shape
    xp = torch.zeros((_ceil(rows, 128) * 128, _ceil(k, 128) * 128), dtype=torch.float64, device=x2.device)
    xp[:rows, :k] = flush_denormals(x2)
    q, e = _quant_last(xp)
    return q[:keep_rows, :keep_cols].contiguous(), atoms(e)


def quant_rows(x: torch.Tensor):
    """``quant_mx_rows``: x [R, C] -> (q [R, round_up(C, 16)] uint8, scale atoms), blocks along C."""
    R, C = x.shape
    return _quant(x, R, _ceil(C, 16) * 16)


def quant_cols(x: torch.Tensor):
    """``quant_mx_cols``: x [R, C] -> (q [C, round_up(R, 16)] uint8 = quantised transpose, scale atoms), blocks
    along R."""
    R, C = x.shape
    return _quant(x.t(), C, _ceil(R, 16) * 16)


def dequant(q: torch.Tensor, sf, K: int) -> torch.Tensor:
    """float64 [rows, K] values of a quantised operand (``sf=None``: unscaled e4m3)."""
    v = decode_e4m3(q[:, :K].contiguous())
    return v if sf is None else v * scales_of(sf, q.shape[0], K)


def gemm(qa, sfa, qb, sfb, K: int, n_valid=None):
    """Block-scaled GEMM ``sum_kb sa * sb * sum_k qa * qb`` in float64, before the epilogue.

    Returns ``(acc, mag)``: ``acc[M, N]`` and ``mag = sum_kb sa * sb * sum_k |qa * qb|``, the size of the terms
    an error bound is proportional to.  ``n_valid`` keeps the first ``n_valid`` columns.  Every product and
    every block sum is exact in float64; only the sum over blocks rounds, at 2^-53."""
    A = dequant(qa, sfa, K)
    B = dequant(qb, sfb, K)
    if n_valid is not None:
        B = B[:n_valid]
    return A @ B.t(), A.abs() @ B.abs().t()


def gelu_tanh(v: torch.Tensor) -> torch.Tensor:
    return 0.5 * v * (1.0 + torch.tanh(math.sqrt(2.0 / math.pi) * (v + 0.044715 * v ** 3)))


def epilogue(acc: torch.Tensor, alpha: float = 1.0, bias=None, act: int = 0, out0=None) -> torch.Tensor:
    """``act(alpha * acc + bias)`` (act 1 = ReLU, 2 = tanh-GELU), added onto ``out0`` when accumulating."""
    v = alpha * acc
    if bias is not None:
        v = v + bias.to(torch.float64)
    if act == 1:
        v = v.clamp_min(0.0)
    elif act == 2:
        v = gelu_tanh(v)
    return v if out0 is None else out0.to(torch.float64) + v
