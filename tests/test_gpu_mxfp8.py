"""MXFP8 quantisers, block-scaled GEMM and fp8 layers against the float64 reference of tests/mxref.py.

The quantisers must reproduce the reference byte for byte: every q byte and every scale byte, padding included.

GEMM error bound.  Every e4m3 product is exact, and the scale fold ``acc += sa * sb * tmp`` multiplies by a power of
two, so only three steps round: the tensor core's sum of one 32-element block, the fp32 fold of the block sums, and
the epilogue.  Hopper's fp8 ``wgmma`` does not add a block in full fp32: it aligns the products and keeps a limited
number of fraction bits (about 14 on H800 by the DeepSeek-V3 report's measurement).  The model used here allows 13:
each of the 32 terms of a block loses at most 2^-13 of the block's sum of magnitudes, so a block is off by at most
32 * 2^-13 = 2^-8 of ``sum |qa * qb|`` times its scales.  The fp32 fold adds at most 2^-23 of the running magnitude per
block.  Hence ``|err| <= (2^-8 + nb * 2^-23) * sum_kb sa * sb * sum |qa * qb|`` with ``nb = ceil(K / 32)``.  The
unscaled kind accumulates the whole K inside ``wgmma``, so each block's add into the accumulator may lose another
2^-13 of the total: ``(2^-8 + nb * 2^-13)``.  fp32 epilogue arithmetic adds 2^-21 of the magnitudes it touches, a bf16
output half an ulp (<= 2^-8 of the value).  Each test prints its worst error / bound ratio (``pytest -rP``).
"""
import math

import pytest
import torch

import mxref

pytestmark = pytest.mark.gpu
BF16 = torch.bfloat16
F32 = torch.float32
DEV = torch.device("cuda:0")


# ---------------------------------------------------------------------------------------------------- helpers
def _same_bytes(got, want, what):
    assert got.shape == want.shape, (what, got.shape, want.shape)
    diff = got != want
    if bool(diff.any()):
        idx = diff.nonzero()[:6]
        pick = tuple(idx.t())
        raise AssertionError("{}: {} of {} bytes differ; first at {}: kernel {} reference {}".format(
            what, int(diff.sum()), diff.numel(), idx.tolist(), got[pick].tolist(), want[pick].tolist()))


def _wide(R, C, seed):
    """bf16 [R, C] whose 32 x 32 blocks have magnitudes from 2^-140 (flushed) up to 2^120."""
    g = torch.Generator().manual_seed(seed)
    exps = torch.arange(-140, 121, 9)
    pick = exps[torch.randint(0, len(exps), (math.ceil(R / 32), math.ceil(C / 32)), generator=g)]
    s = pick.repeat_interleave(32, 0)[:R].repeat_interleave(32, 1)[:, :C].double()
    return (torch.randn(R, C, generator=g, dtype=torch.float64) * torch.exp2(s)).to(BF16).to(DEV)


def _operand(R, C, seed, along=1, spread=3):
    """bf16 [R, C], every 32-element block along ``along`` scaled by its own 2^[-spread, spread]: adjacent rows and
    blocks get different scale bytes, in a range where no scale product can underflow."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    shape = (R, math.ceil(C / 32)) if along == 1 else (math.ceil(R / 32), C)
    s = torch.randint(-spread, spread + 1, shape, generator=g, device=DEV).float()
    s = s.repeat_interleave(32, along)[:R, :C]
    return (torch.randn(R, C, generator=g, device=DEV) * torch.exp2(s)).to(BF16)


def _c(K, scaled=True):
    nb = math.ceil(K / 32)
    return 2.0 ** -8 + nb * (2.0 ** -23 if scaled else 2.0 ** -13)


def _tol(mag, K, *, want, alpha=1.0, bias=None, act=0, out0=None, bf16=False, scaled=True):
    """Per-element bound on |kernel - reference| (see the module docstring)."""
    t = abs(alpha) * _c(K, scaled) * mag
    touched = abs(alpha) * mag
    if bias is not None:
        touched = touched + bias.double().abs()
    if out0 is not None:
        touched = touched + out0.double().abs()
    t = t + 2.0 ** -21 * touched
    if act == 2:        # tanh-GELU is 1.13-Lipschitz; tanhf and the cubic add a few fp32 ulps of the argument
        t = 1.13 * t + 2.0 ** -20 * touched
    if bf16:
        t = t + 2.0 ** -8 * (want.abs() + t)
    return t


def _check(family, got, want, tol):
    got = got.detach().double()
    err = (got - want).abs()
    ratio = float((err / tol.clamp_min(1e-300)).max())
    print("worst error/bound {}: {:.4g}".format(family, ratio))
    bad = ~(err <= tol)
    if bool(bad.any()):
        idx = bad.nonzero()[:5]
        pick = tuple(idx.t())
        raise AssertionError("{}: {} of {} elements out of bound; first at {}: kernel {} reference {} bound {}".format(
            family, int(bad.sum()), bad.numel(), idx.tolist(), got[pick].tolist(), want[pick].tolist(),
            tol[pick].tolist()))


# ---------------------------------------------------------------------------------------------------- quantisers
# (R, C, row pitch): ragged R and C, partial 32-row tiles of the transposed store (round_up(R, 16) % 32 == 16),
# pitches with ld % 8 == 0 (vector loads) and ld % 8 != 0 (scalar loads); views are sliced from column 0
QUANT_CASES = [(256, 512, 512), (300, 200, 200), (128, 4608, 4608), (1000, 72, 72),
               (300, 200, 208), (300, 200, 203), (257, 33, 40), (257, 33, 35), (4100, 160, 168), (16, 40, 45),
               (48, 4104, 4104)]


@pytest.mark.parametrize("R,C,ld", QUANT_CASES)
def test_quant_rows_bytes_match_reference(R, C, ld):
    from baton_b200.ops import functional as F
    x = _wide(R, ld, R * 3 + ld)[:, :C]
    q, sf = F.quant_mx_rows(x)
    rq, rsf = mxref.quant_rows(x)
    _same_bytes(sf, rsf, "scale bytes")
    _same_bytes(q, rq, "q bytes")


@pytest.mark.parametrize("R,C,ld", QUANT_CASES)
def test_quant_cols_bytes_match_reference(R, C, ld):
    from baton_b200.ops import functional as F
    x = _wide(R, ld, R * 5 + ld)[:, :C]
    q, sf = F.quant_mx_cols(x)
    rq, rsf = mxref.quant_cols(x)
    _same_bytes(sf, rsf, "scale bytes")
    _same_bytes(q, rq, "q bytes")


def test_quant_inf_and_nan_today():
    """+-inf saturates to a finite +-448 * 2^120 (the exponent field of inf gives e = 120); NaN is skipped in amax
    and stays NaN (0x7F); a block of NaN only gets scale byte 0."""
    from baton_b200.ops import functional as F
    inf, nan = float("inf"), float("nan")
    x = torch.randn(64, 96, device=DEV).to(BF16)
    x[0, :3] = torch.tensor([inf, -inf, nan])
    x[1, 32:64] = nan
    x[5, 70] = nan
    x[40, 3] = inf
    for quant, ref in ((F.quant_mx_rows, mxref.quant_rows), (F.quant_mx_cols, mxref.quant_cols)):
        q, sf = quant(x)
        rq, rsf = ref(x)
        _same_bytes(sf, rsf, quant.__name__ + " scale bytes")
        _same_bytes(q, rq, quant.__name__ + " q bytes")
    q, sf = F.quant_mx_rows(x)
    assert q[0, :3].tolist() == [0x7E, 0xFE, 0x7F]
    assert q[1, 32:64].tolist() == [0x7F] * 32
    assert int(sf[0]) == 120 + 127                      # row 0, block 0 (offset 0 of atom 0)
    assert int(sf[1 * 16 + 1]) == 0                     # row 1, block 1
    # NaN skipped: row 5, block 2 has the scale of its finite elements
    fin = x[5, 64:96].float().abs().nan_to_num(0.0).amax()
    assert int(sf[5 * 16 + 2]) - 127 == int(mxref.block_exponent(fin.double().view(1))[0])


# ---------------------------------------------------------------------------------------------------- GEMM
# ResNet-18 / ResNet-50 layers at batch 128 on 32 x 32 inputs (M x N x K), the stem forward (K = 147 padded to 152),
# and the shapes of the earlier dequantise-and-matmul test
GEMM_SHAPES = [(8192, 64, 576), (8192, 256, 64), (2048, 128, 1152), (512, 256, 2304), (512, 1024, 256),
               (128, 512, 4608), (128, 2048, 512), (32768, 64, 152),
               (128, 128, 128), (256, 384, 512), (300, 200, 1000), (512, 64, 4608), (1000, 256, 72)]
_CASES = {}


def _gemm_case(M, N, K):
    """Kernel operands from the project's quantisers; reference from mxref's quantisers of the same bf16 inputs."""
    key = (M, N, K)
    if key not in _CASES:
        from baton_b200.ops import functional as F
        A, B = _operand(M, K, 7 * M + K), _operand(N, K, 13 * N + K + 1)
        qa, sa = F.quant_mx_rows(A)
        qb, sb = F.quant_mx_rows(B)
        acc, mag = mxref.gemm(*mxref.quant_rows(A), *mxref.quant_rows(B), K)
        _CASES.clear()
        _CASES[key] = (qa, sa, qb, sb, acc, mag)
    return _CASES[key]


@pytest.mark.parametrize("M,N,K", GEMM_SHAPES)
def test_gemm_matches_reference(M, N, K):
    from baton_b200.ops import functional as F
    qa, sa, qb, sb, acc, mag = _gemm_case(M, N, K)
    out = F.gemm_fp8(qa, sa, qb, sb, K, out_dtype=F32)
    assert out.shape == (M, N)
    _check("fp32", out, acc, _tol(mag, K, want=acc))
    out = F.gemm_fp8(qa, sa, qb, sb, K)
    assert out.dtype == BF16
    _check("bf16", out, acc, _tol(mag, K, want=acc, bf16=True))


@pytest.mark.parametrize("M,N,K", [(300, 200, 1000), (1000, 256, 72), (512, 1024, 256), (8192, 64, 576)])
def test_gemm_epilogue(M, N, K):
    from baton_b200.ops import functional as F
    qa, sa, qb, sb, acc, mag = _gemm_case(M, N, K)
    g = torch.Generator(device=DEV).manual_seed(M + N)
    alpha = 0.75 / float(acc.std())                    # puts most of the GELU inputs in its curved region
    bias = torch.randn(N, generator=g, device=DEV)
    for fam, kw, bf16 in (("bias+relu", dict(bias=bias, act=1), True),
                          ("bias+gelu", dict(bias=bias, act=2, alpha=alpha), False),
                          ("gelu", dict(act=2, alpha=-alpha), True)):
        out = F.gemm_fp8(qa, sa, qb, sb, K, out_dtype=BF16 if bf16 else F32, **kw)
        want = mxref.epilogue(acc, kw.get("alpha", 1.0), kw.get("bias"), kw["act"])
        _check(fam, out, want, _tol(mag, K, want=want, alpha=kw.get("alpha", 1.0), bias=kw.get("bias"), act=kw["act"],
                                    bf16=bf16))
    out = F.gemm_fp8(qa, sa, qb, sb, K, out_dtype=F32, alpha=alpha)
    _check("alpha", out, alpha * acc, _tol(mag, K, want=acc, alpha=alpha))


@pytest.mark.parametrize("accumulate", [False, True])
@pytest.mark.parametrize("split_k", [2, 3, 7])
@pytest.mark.parametrize("M,N,K", [(300, 200, 1000), (512, 64, 4608), (128, 512, 4608), (2048, 128, 1152)])
def test_gemm_split_k(M, N, K, split_k, accumulate):
    from baton_b200.ops import functional as F
    qa, sa, qb, sb, acc, mag = _gemm_case(M, N, K)
    if accumulate:
        g = torch.Generator(device=DEV).manual_seed(split_k)
        out0 = torch.randn(M, N, generator=g, device=DEV) * float(acc.std())
        out = out0.clone()
        F.gemm_fp8(qa, sa, qb, sb, K, out=out, accumulate=True, split_k=split_k)
        _check("accumulate", out, out0.double() + acc, _tol(mag, K, want=acc, out0=out0))
    else:
        out = F.gemm_fp8(qa, sa, qb, sb, K, out_dtype=F32, split_k=split_k)
        _check("split_k", out, acc, _tol(mag, K, want=acc))
        out = torch.full((M, N), float("nan"), device=DEV)
        F.gemm_fp8(qa, sa, qb, sb, K, out=out, split_k=split_k)          # a given output is overwritten, too
        _check("split_k", out, acc, _tol(mag, K, want=acc))


def test_gemm_split_k_output_starts_from_zero():
    """Split-K adds its slices with atomics: an output taken from the caching allocator must be zeroed first.  The
    block freed just before holds NaN, so a missing zero-fill shows on every element."""
    from baton_b200.ops import functional as F
    M, N, K = 300, 200, 1000
    qa, sa, qb, sb, acc, mag = _gemm_case(M, N, K)
    junk = torch.full((M, N), float("nan"), device=DEV)
    addr = junk.data_ptr()
    del junk
    out = F.gemm_fp8(qa, sa, qb, sb, K, out_dtype=F32, split_k=3)
    assert out.data_ptr() == addr, "the allocator did not hand back the NaN block; the test proves nothing"
    _check("split_k", out, acc, _tol(mag, K, want=acc))


def test_gemm_pitched_outputs():
    """Outputs in a wider buffer: fp32 and bf16 stores at pitches that do and do not allow 16-byte vectors, ragged
    N; the columns past N stay untouched."""
    from baton_b200.ops import functional as F
    M, N, K = 300, 200, 1000
    qa, sa, qb, sb, acc, mag = _gemm_case(M, N, K)
    for dtype, pad in ((F32, 1), (F32, 4), (BF16, 8), (BF16, 3)):
        buf = torch.full((M, N + pad), -7.0, dtype=dtype, device=DEV)
        out = buf[:, :N]
        F.gemm_fp8(qa, sa, qb, sb, K, out=out)
        _check("bf16" if dtype == BF16 else "fp32", out, acc, _tol(mag, K, want=acc, bf16=dtype == BF16))
        assert bool((buf[:, N:] == -7.0).all()), "store past N at pitch {}".format(N + pad)


def test_gemm_wgrad_n_valid():
    """The stem's weight gradient: dW[64, 147] += dY^T X over 32768 rows, B padded to 152 rows (K of the stem padded
    147 -> 152), into a 147-wide gradient and into a pitched one."""
    from baton_b200.ops import functional as F
    Mr, N, Kp, nv = 32768, 64, 152, 147
    dy = _operand(Mr, N, 1, along=0)
    col = _operand(Mr, Kp, 2, along=0)
    col[:, nv:] = 0
    dyt, sdyt = F.quant_mx_cols(dy)
    xt, sxt = F.quant_mx_cols(col)
    acc, mag = mxref.gemm(*mxref.quant_cols(dy), *mxref.quant_cols(col), Mr, n_valid=nv)
    assert acc.shape == (N, nv)
    g0 = torch.randn(N, nv, device=DEV) * float(acc.std())
    out = g0.clone()
    F.gemm_fp8(dyt, sdyt, xt, sxt, Mr, out=out, accumulate=True, n_valid=nv)
    _check("n_valid", out, g0.double() + acc, _tol(mag, Mr, want=acc, out0=g0))
    buf = torch.full((N, 160), -7.0, device=DEV)
    buf[:, :nv] = g0
    F.gemm_fp8(dyt, sdyt, xt, sxt, Mr, out=buf[:, :nv], accumulate=True, n_valid=nv)
    _check("n_valid", buf[:, :nv], g0.double() + acc, _tol(mag, Mr, want=acc, out0=g0))
    assert bool((buf[:, nv:] == -7.0).all())
    out = F.gemm_fp8(dyt, sdyt, xt, sxt, Mr, out_dtype=F32, n_valid=nv)
    assert out.shape == (N, nv)
    _check("n_valid", out, acc, _tol(mag, Mr, want=acc))


@pytest.mark.parametrize("N,K", [(64, 512), (40, 272), (64, 4608)])
def test_gemm_unscaled_bn64(N, K):
    """The unscaled kind at N <= 64 runs the BN = 64 instantiation."""
    from baton_b200.ops import functional as F
    g = torch.Generator(device=DEV).manual_seed(N + K)
    M = 300
    qa = (torch.randn(M, K, generator=g, device=DEV) * 2).clamp(-400, 400).to(torch.float8_e4m3fn).view(torch.uint8)
    qb = torch.randn(N, K, generator=g, device=DEV).to(torch.float8_e4m3fn).view(torch.uint8)
    acc, mag = mxref.gemm(qa, None, qb, None, K)
    out = F.gemm_fp8(qa, None, qb, None, K, out_dtype=F32, alpha=0.5)
    _check("unscaled", out, 0.5 * acc, _tol(mag, K, want=acc, alpha=0.5, scaled=False))
    out = F.gemm_fp8(qa, None, qb, None, K, alpha=0.5)
    _check("unscaled", out, 0.5 * acc, _tol(mag, K, want=0.5 * acc, alpha=0.5, scaled=False, bf16=True))


# ---------------------------------------------------------------------------------------------------- layers
def _im2col(x, k, s, p, kp):
    """NHWC bf16 -> float64 col [N*Ho*Wo, kp], columns ordered (kh, kw, c) like the OHWI weights, zero past k*k*c."""
    n, h, w, c = x.shape
    cols = torch.nn.functional.unfold(x.double().permute(0, 3, 1, 2), k, padding=p, stride=s)   # [n, c*k*k, L]
    L = cols.shape[-1]
    out = torch.zeros(n * L, kp, dtype=torch.float64, device=x.device)
    out[:, : k * k * c] = cols.view(n, c, k * k, L).permute(0, 3, 2, 1).reshape(n * L, k * k * c)
    return out


def _col2im(dcol, shape, k, s, p):
    n, h, w, c = shape
    ho, wo = (h + 2 * p - k) // s + 1, (w + 2 * p - k) // s + 1
    t = dcol[:, : k * k * c].reshape(n, ho * wo, k * k, c).permute(0, 3, 2, 1).reshape(n, c * k * k, ho * wo)
    return torch.nn.functional.fold(t, (h, w), k, padding=p, stride=s).permute(0, 2, 3, 1)


def _grad2d(weight):
    """The [Cout, K] view of a weight gradient (OHWI for a channels-last conv weight)."""
    g = weight.grad
    return g.permute(0, 2, 3, 1).reshape(g.shape[0], -1) if g.dim() == 4 else g


def _layer_refs(col, wb, dy2, k_true):
    """y = Q_rows(col) Q_rows(w)^T, dcol = Q_rows(dy) Q_cols(w), dW = Q_cols(dy)^T Q_cols(col): (acc, mag) each."""
    K, N = col.shape[1], wb.shape[0]
    y = mxref.gemm(*mxref.quant_rows(col), *mxref.quant_rows(wb), K)
    dcol = mxref.gemm(*mxref.quant_rows(dy2), *mxref.quant_cols(wb), N)
    dw = mxref.gemm(*mxref.quant_cols(dy2), *mxref.quant_cols(col), col.shape[0], n_valid=k_true)
    return y, dcol, dw


def _check_layer(y2, dy2, col, wb, k_true, gw, g0, dx_fn=None, dx=None):
    (ya, ym), (da, dm), (wa, wm) = _layer_refs(col, wb, dy2, k_true)
    _check("layer y", y2, ya, _tol(ym, col.shape[1], want=ya, bf16=True))
    _check("layer dW", gw, g0.double() + wa, _tol(wm, col.shape[0], want=wa, out0=g0))
    if dx is not None:
        t = _tol(dm, wb.shape[0], want=da, bf16=True)          # dcol is stored in bf16 ...
        want = dx_fn(da)
        t = dx_fn(t)                                           # ... and col2im adds up to k*k of them
        _check("layer dx", dx, want, t + 2.0 ** -8 * (want.abs() + t) + 2.0 ** -21 * dx_fn(da.abs()))


CONV_CASES = [  # (cin, cout, k, stride, pad, n, h): rows n*Ho*Wo = 75, 100, 75, 450 (none a multiple of 16 but 450)
    (64, 128, 3, 1, 1, 3, 5), (64, 128, 3, 2, 1, 4, 9), (128, 256, 1, 1, 0, 3, 5), (3, 64, 7, 2, 3, 2, 30)]


@pytest.mark.parametrize("arena", [False, True])
@pytest.mark.parametrize("cin,cout,k,stride,pad,n,h", CONV_CASES)
def test_conv2d_fp8_matches_reference(cin, cout, k, stride, pad, n, h, arena):
    from baton_b200.ops import nn as bnn
    from baton_b200.parallel.arena import ParamArena
    torch.manual_seed(cin + k + stride + n)
    conv = bnn.Conv2d(cin, cout, k, stride, pad).to(DEV)
    k_true, kp = conv.k_true, conv.kp
    ar = ParamArena(conv, DEV) if arena else None
    conv.fp8 = True
    wb = torch.zeros(cout, kp, dtype=BF16, device=DEV)
    wb[:, :k_true] = conv.weight.detach().permute(0, 2, 3, 1).reshape(cout, k_true).to(BF16)
    needs_dx = cin % 8 == 0                               # the C = 3 stem has no input gradient
    x = torch.randn(n, h, h, cin, device=DEV).to(BF16).requires_grad_(needs_dx)
    col = _im2col(x.detach(), k, stride, pad, kp)
    shape = tuple(x.shape)
    fold = (lambda d: d.view(shape)) if k == 1 else (lambda d: _col2im(d, shape, k, stride, pad))
    g0 = None
    if arena:
        ar.grad.copy_(torch.randn_like(ar.grad))
        g0 = _grad2d(conv.weight).clone()
    for step in range(1 if arena else 2):                 # outside an arena: first into no gradient, then onto it
        if not arena:
            g0 = torch.zeros(cout, k_true, device=DEV) if step == 0 else _grad2d(conv.weight).clone()
        x.grad = None
        y = conv(x)
        assert y.dtype == BF16 and y.shape[:3] == (n, (h + 2 * pad - k) // stride + 1, (h + 2 * pad - k) // stride + 1)
        dy = torch.randn_like(y)
        y.backward(dy)
        _check_layer(y.reshape(-1, cout), dy.reshape(-1, cout), col, wb, k_true, _grad2d(conv.weight), g0,
                     fold, x.grad if needs_dx else None)
        if needs_dx:
            assert x.grad is not None


@pytest.mark.parametrize("arena", [False, True])
def test_linear_fp8_matches_reference(arena):
    from baton_b200.ops import nn as bnn
    from baton_b200.parallel.arena import ParamArena
    torch.manual_seed(11)
    M, K, N = 300, 576, 256
    lin = bnn.Linear(K, N, bias=False).to(DEV)
    ar = ParamArena(lin, DEV) if arena else None
    lin.fp8 = True
    wb = lin.weight.detach().to(BF16)
    x = torch.randn(M, K, device=DEV).to(BF16).requires_grad_(True)
    col = x.detach().double()
    g0 = None
    if arena:
        ar.grad.copy_(torch.randn_like(ar.grad))
        g0 = lin.weight.grad.clone()
    for step in range(1 if arena else 2):
        if not arena:
            g0 = torch.zeros(N, K, device=DEV) if step == 0 else lin.weight.grad.clone()
        x.grad = None
        y = lin(x)
        dy = torch.randn_like(y)
        y.backward(dy)
        _check_layer(y, dy, col, wb, K, lin.weight.grad, g0, lambda d: d, x.grad)


def test_conv2d_fp8_cuda_graph_replay_is_bitwise_eager():
    """Forward and backward of an fp8 convolution captured in a CUDA graph replay the eager result bit for bit.  The
    capture includes the weight-gradient accumulate, so the gradient is reset before each replay; with split_k = 1
    each gradient element gets one atomic add, so the result is deterministic."""
    from baton_b200.ops import nn as bnn
    from baton_b200.parallel.arena import ParamArena
    torch.manual_seed(5)
    conv = bnn.Conv2d(64, 128, 3, 1, 1).to(DEV)
    ar = ParamArena(conv, DEV)
    conv.fp8 = True
    x = torch.randn(4, 8, 8, 64, device=DEV).to(BF16)
    dy = torch.randn(4, 8, 8, 128, device=DEV).to(BF16)

    def step():
        # a fresh leaf over the same storage: autograd's node for it then lives on the stream being captured
        xl = x.detach().requires_grad_(True)
        y = conv(xl)
        dx, = torch.autograd.grad(y, xl, dy)
        return y.detach(), dx

    ar.grad.zero_()
    y_e, dx_e = step()
    g_e = ar.grad.clone()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        step()
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        y_g, dx_g = step()
    for _ in range(2):
        ar.grad.zero_()
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(y_g, y_e) and torch.equal(dx_g, dx_e) and torch.equal(ar.grad, g_e)
