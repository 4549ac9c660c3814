"""The MXFP8 reference (tests/mxref.py) against hand-worked cases of the format.  CPU only: the GPU tests of the
quantisers and the fp8 GEMM trust this module, so it is checked here byte by byte."""
import itertools
import math

import pytest
import torch

import mxref

BF16 = torch.bfloat16


def _block(*vals):
    """One row of one 32-element block: ``vals`` first, zeros after."""
    x = torch.zeros(1, 32, dtype=torch.float64)
    x[0, : len(vals)] = torch.tensor(vals, dtype=torch.float64)
    assert torch.equal(x.to(BF16).double(), x), "hand-worked inputs must be exact in bf16"
    return x.to(BF16)


def _one(*vals):
    q, sf = mxref.quant_rows(_block(*vals))
    return int(sf[0]) - 127, q[0, : len(vals)].tolist()


def test_exponent_at_and_just_above_mantissa_1_75():
    # 1.75 * 2^3 = 14: floor(log2) = 3, no bump, e = -5, and 14 * 2^5 = 448 = 0x7E exactly
    assert _one(14.0) == (-5, [0x7E])
    # 1.7578125 * 2^3 (the next bf16): bumped to e = -4; 225 rounds to 224 = 1.75 * 2^7 = 0x76
    assert _one(1.7578125 * 8) == (-4, [0x76])
    # 1.5 * 2^3: no bump, 12 * 2^5 = 384 = 1.5 * 2^8 = 0x7C
    assert _one(12.0) == (-5, [0x7C])


def test_bf16_maximum():
    big = float(torch.finfo(BF16).max)                  # (2 - 2^-7) * 2^127, mantissa above 1.75
    e, q = _one(big, -big, 1.0)
    assert e == 120
    # big * 2^-120 = 254 rounds to 256 = 2^8 (0x78); 1.0 * 2^-120 is far below the smallest e4m3 subnormal
    assert q == [0x78, 0xF8, 0x00]


def test_bf16_subnormals_flush_to_zero():
    tiny = 2.0 ** -130                                  # a bf16 subnormal: flushed in amax and as an element
    assert _one(tiny, -tiny) == (-127, [0x00, 0x80])
    # the smallest normal is kept: e = -126 - 8 clamps to -127, and 2^-126 * 2^127 = 2 = 0x40
    assert _one(2.0 ** -126, tiny) == (-127, [0x40, 0x00])
    q, sf = mxref.quant_rows(_block(tiny))
    assert mxref.scales_of(sf, 1, 32)[0, 0] == 0.0     # the GEMM decodes scale byte 0 as 0, not 2^-127


def test_e4m3_subnormals_and_ties_round_to_even():
    # amax 1.0: e = -8, elements are scaled by 2^8; the e4m3 subnormal step is 2^-9
    u = 2.0 ** -17                                      # 2^-9 after scaling
    e, q = _one(1.0, u, 1.5 * u, 0.5 * u, 2.5 * u, 1.0625 * 2 ** -8, 1.1875 * 2 ** -8, -1.5 * u)
    assert e == -8
    assert q == [0x78,          # 1.0 * 2^8 = 256
                 0x01,          # smallest subnormal
                 0x02,          # 1.5 steps: tie, to the even 2 steps
                 0x00,          # half a step: tie, to zero
                 0x02,          # 2.5 steps: tie, to 2
                 0x38,          # 1.0625: tie between 1.0 (0x38) and 1.125 (0x39), to 0x38
                 0x3A,          # 1.1875: tie between 1.125 and 1.25 (0x3A), to 0x3A
                 0x82]          # sign of a subnormal


def test_all_zero_block():
    q, sf = mxref.quant_rows(torch.zeros(3, 70, dtype=BF16))
    assert q.shape == (3, 80) and int(q.count_nonzero()) == 0
    assert sf.shape == (512,) and int(sf.count_nonzero()) == 0


def test_inf_and_nan():
    inf, nan = float("inf"), float("nan")
    x = torch.zeros(2, 64, dtype=BF16)
    x[0, :4] = torch.tensor([inf, 1.0, nan, -inf])
    x[0, 32:34] = torch.tensor([nan, 0.5])              # NaN is skipped in amax: e = -9
    x[1, :32] = nan                                      # all NaN: amax 0
    q, sf = mxref.quant_rows(x)
    e = mxref.scales_of(sf, 2, 64)[:, ::32].log2()
    assert e[0].tolist() == [120.0, -9.0]               # +-inf counts as 2^128
    assert mxref.scales_of(sf, 2, 64)[1, 0] == 0.0      # byte 0
    assert q[0, :4].tolist() == [0x7E, 0x00, 0x7F, 0xFE]
    assert q[0, 32:34].tolist() == [0x7F, 0x78]         # 0.5 * 2^9 = 256
    assert q[1, :32].tolist() == [0x7F] * 32


def _wide(R, C, seed):
    """bf16 [R, C] whose 32 x 32 blocks have magnitudes from 2^-140 (flushed) to 2^120."""
    g = torch.Generator().manual_seed(seed)
    exps = torch.arange(-140, 121, 9)
    pick = exps[torch.randint(0, len(exps), (math.ceil(R / 32), math.ceil(C / 32)), generator=g)]
    s = pick.repeat_interleave(32, 0)[:R].repeat_interleave(32, 1)[:, :C].double()
    return (torch.randn(R, C, generator=g, dtype=torch.float64) * torch.exp2(s)).to(BF16)


@pytest.mark.parametrize("R,C", [(37, 200), (130, 72), (256, 512)])
def test_decoded_elements_within_half_a_step(R, C):
    x = _wide(R, C, R + C)
    q, sf = mxref.quant_rows(x)
    back = mxref.dequant(q, sf, C)
    xf = mxref.flush_denormals(x)
    scale = mxref.scales_of(sf, R, C)
    # scale 0 (byte 0) only where the whole block is below 2^-119
    assert bool((xf.abs()[scale == 0] < 2.0 ** -118).all())
    ok = scale > 0
    v = xf / torch.where(ok, scale, torch.ones_like(scale))        # the element in units of its block scale
    step = torch.exp2(torch.floor(torch.log2(v.abs().clamp_min(2.0 ** -6))) - 3)   # e4m3 spacing (2^-9 subnormal)
    err = (back - xf).abs() / torch.where(ok, scale, torch.ones_like(scale))
    assert bool((err[ok] <= step[ok] / 2).all())
    # the block maximum lands in (224, 448]: it never saturates and the scale never wastes the top binade
    vp = torch.zeros(R, math.ceil(C / 32) * 32, dtype=torch.float64)
    vp[:, :C] = v.abs()
    amax = vp.view(R, -1, 32).amax(-1)
    live = ok[:, ::32]
    assert bool(((amax[live] > 224) & (amax[live] <= 448)).all())


def _sf_offset(row, k, k_tiles):           # the index formula at the top of csrc/quant.cu, written out
    return ((row >> 7) * k_tiles + (k >> 7)) * 512 + (row & 31) * 16 + ((row & 127) >> 5) * 4 + ((k & 127) >> 5)


def test_atom_layout_matches_index_formula():
    R, C = 200, 300
    x = _wide(R, C, 5)
    q, sf = mxref.quant_rows(x)
    Rpad, Cpad = 256, 384
    assert sf.numel() == (Rpad // 128) * (Cpad // 128) * 512
    assert q.shape == (R, 304)
    xp = torch.zeros(Rpad, Cpad, dtype=torch.float64)
    xp[:R, :C] = mxref.flush_denormals(x)
    seen = torch.zeros_like(sf, dtype=torch.bool)
    for r, kb in itertools.product(range(Rpad), range(Cpad // 32)):
        blk = xp[r, 32 * kb: 32 * kb + 32]
        amax = float(blk.abs().max())
        want = 0 if amax == 0 else max(-127, min(127, math.frexp(amax)[1] - 1 - 8 + (2 * math.frexp(amax)[0] > 1.75))) + 127
        off = _sf_offset(r, 32 * kb, Cpad // 128)
        assert int(sf[off]) == want, (r, kb)
        seen[off] = True
    assert bool(seen.all())                             # every byte of the buffer, padding atoms included


def test_cols_is_rows_of_the_transpose():
    x = _wide(300, 70, 9)
    q, sf = mxref.quant_cols(x)
    qt, sft = mxref.quant_rows(x.t().contiguous())
    assert q.shape == (70, 304)
    assert torch.equal(q[:, :300], qt[:, :300]) and int(q[:, 300:].count_nonzero()) == 0
    assert torch.equal(sf, sft)


@pytest.mark.parametrize("n_valid", [None, 37])
def test_gemm_is_the_blockwise_sum(n_valid):
    g = torch.Generator().manual_seed(2)
    M, N, K = 5, 40, 100
    A = (torch.randn(M, K, generator=g) * torch.exp2(torch.randint(-3, 4, (M, K), generator=g).float())).to(BF16)
    B = (torch.randn(N, K, generator=g) * torch.exp2(torch.randint(-3, 4, (N, K), generator=g).float())).to(BF16)
    qa, sa = mxref.quant_rows(A)
    qb, sb = mxref.quant_rows(B)
    acc, mag = mxref.gemm(qa, sa, qb, sb, K, n_valid=n_valid)
    n = N if n_valid is None else n_valid
    assert acc.shape == (M, n)
    va, vb = mxref.decode_e4m3(qa), mxref.decode_e4m3(qb)
    for m, j in itertools.product(range(M), range(n)):
        want = wmag = 0.0
        for kb in range(math.ceil(K / 32)):
            sab = 2.0 ** (int(sa[_sf_offset(m, 32 * kb, 1)]) - 127) * 2.0 ** (int(sb[_sf_offset(j, 32 * kb, 1)]) - 127)
            ks = slice(32 * kb, min(K, 32 * kb + 32))
            want += sab * float((va[m, ks] * vb[j, ks]).sum())
            wmag += sab * float((va[m, ks] * vb[j, ks]).abs().sum())
        assert math.isclose(float(acc[m, j]), want, rel_tol=1e-14, abs_tol=1e-300)
        assert math.isclose(float(mag[m, j]), wmag, rel_tol=1e-14)
    # it approximates the bf16 product to within the e4m3 rounding of both operands
    exact = A.double() @ B.double()[:n].t()
    bound = (A.double().abs() @ B.double()[:n].abs().t()) * (2 * 2.0 ** -4 + 2.0 ** -8)
    assert bool(((acc - exact).abs() <= bound).all())


def test_epilogue():
    acc = torch.tensor([[-2.0, 0.0, 3.0]], dtype=torch.float64)
    bias = torch.tensor([1.0, -1.0, 0.5])
    assert mxref.epilogue(acc, 0.5, bias, act=1).tolist() == [[0.0, 0.0, 2.0]]
    v = mxref.epilogue(acc, 1.0, None, act=2)
    want = [0.5 * a * (1 + math.tanh(math.sqrt(2 / math.pi) * (a + 0.044715 * a ** 3))) for a in (-2.0, 0.0, 3.0)]
    assert v[0].tolist() == pytest.approx(want, rel=1e-15)
    assert mxref.epilogue(acc, 2.0, out0=torch.ones(1, 3)).tolist() == [[-3.0, 1.0, 7.0]]
