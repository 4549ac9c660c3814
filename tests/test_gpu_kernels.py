"""Kernel-correctness tier: every sm_90a kernel against a plain PyTorch fp32
reference of the same op (SURVEY.md section 4)."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

BF16 = torch.bfloat16


def _dev():
    return torch.device("cuda:0")


def _rel(a, b):
    a, b = a.float(), b.float()
    return float((a - b).abs().max() / (b.abs().max() + 1e-6))


@pytest.fixture(scope="module")
def F():
    from baton_b200.ops import functional
    return functional


@pytest.fixture(scope="module")
def bnn():
    from baton_b200.ops import nn
    return nn


# ------------------------------------------------------------------ GEMM
@pytest.mark.parametrize("a_mn,b_mn", [(False, False), (False, True), (True, False), (True, True)])
@pytest.mark.parametrize("M,N,K", [(128, 128, 64), (256, 512, 576), (384, 200, 1000), (100, 64, 72), (1000, 1000, 4096)])
def test_gemm_tcgen05_all_majors(F, a_mn, b_mn, M, N, K):
    torch.manual_seed(M + N + K)
    dev = _dev()
    if (a_mn and M % 8) or (b_mn and N % 8) or K % 8:
        pytest.skip("pitch not TMA aligned for this combination")
    A = torch.randn(M, K, device=dev).to(BF16)
    B = torch.randn(N, K, device=dev).to(BF16)
    a = A.t().contiguous() if a_mn else A
    b = B.t().contiguous() if b_mn else B
    ref = A.float() @ B.float().t()
    out = F.gemm(a, b, a_mn=a_mn, b_mn=b_mn, out_dtype=torch.float32)
    assert out.shape == (M, N)
    assert _rel(out, ref) < 2e-3, _rel(out, ref)
    out16 = F.gemm(a, b, a_mn=a_mn, b_mn=b_mn)
    assert out16.dtype == BF16 and _rel(out16, ref) < 1e-2


@pytest.mark.parametrize("bn", [64, 128])     # the host clamps a requested 256 to 128: no 256-wide kernel exists
def test_gemm_tile_widths_bias_act(F, bn):
    torch.manual_seed(bn)
    dev = _dev()
    M, N, K = 300, 520, 328
    A = torch.randn(M, K, device=dev).to(BF16)
    B = torch.randn(N, K, device=dev).to(BF16)
    bias = torch.randn(N, device=dev)
    ref = torch.relu(0.5 * (A.float() @ B.float().t()) + bias)
    out = F.gemm(A, B, bias=bias, act=1, alpha=0.5, out_dtype=torch.float32, force_bn=bn)
    assert _rel(out, ref) < 2e-3
    refg = torch.nn.functional.gelu(A.float() @ B.float().t() + bias, approximate="tanh")
    outg = F.gemm(A, B, bias=bias, act=2, out_dtype=torch.float32, force_bn=bn)
    assert _rel(outg, refg) < 2e-3


def test_gemm_split_k_accumulate_and_pitched_output(F):
    torch.manual_seed(1)
    dev = _dev()
    M, N, K = 64, 576, 16384          # wgrad-like: few tiles, long K
    A = torch.randn(K, M, device=dev).to(BF16)     # MN-major operands
    B = torch.randn(K, N, device=dev).to(BF16)
    ref = A.float().t() @ B.float()
    out = torch.zeros(M, N, device=dev)
    F.gemm(A, B, a_mn=True, b_mn=True, out=out, accumulate=True)
    assert _rel(out, ref) < 2e-3
    F.gemm(A, B, a_mn=True, b_mn=True, out=out, accumulate=True, split_k=7)
    assert _rel(out, 2 * ref) < 2e-3
    # n_valid + narrower output pitch (conv stem: K padded 147 -> 152)
    Bp = torch.zeros(K, 152, device=dev, dtype=BF16)
    Bp[:, :147] = torch.randn(K, 147, device=dev).to(BF16)
    out2 = torch.zeros(M, 147, device=dev)
    F.gemm(A, Bp, a_mn=True, b_mn=True, out=out2, accumulate=True, n_valid=147)
    assert _rel(out2, A.float().t() @ Bp[:, :147].float()) < 2e-3


@pytest.mark.parametrize("S", [2, 4, 8])
@pytest.mark.parametrize("M,N,K,bn", [(128, 512, 4608, 64), (512, 256, 2304, 64), (200, 136, 1032, 128), (256, 512, 2048, 256)])
def test_gemm_cluster_split_k_dsmem_reduce(F, S, M, N, K, bn):
    """Split-K whose z-slices form a thread-block cluster and reduce through distributed smem."""
    torch.manual_seed(S + M)
    dev = _dev()
    A = torch.randn(M, K, device=dev).to(BF16)
    B = torch.randn(N, K, device=dev).to(BF16)
    bias = torch.randn(N, device=dev)
    ref = torch.relu(A.float() @ B.float().t() + bias)
    out = F.gemm(A, B, bias=bias, act=1, split_k=-S, force_bn=bn)
    assert out.dtype == BF16 and _rel(out, ref) < 1e-2, _rel(out, ref)
    out32 = F.gemm(A, B, bias=bias, act=1, split_k=-S, force_bn=bn, out_dtype=torch.float32)
    assert _rel(out32, ref) < 2e-3
    # MN-major operands + accumulate into an existing fp32 buffer
    acc = torch.ones(M, N, device=dev)
    F.gemm(A.t().contiguous(), B.t().contiguous(), a_mn=True, b_mn=True, out=acc, accumulate=True, split_k=-S,
           force_bn=bn) if M % 8 == 0 and N % 8 == 0 else None
    if M % 8 == 0 and N % 8 == 0:
        assert _rel(acc, A.float() @ B.float().t() + 1.0) < 2e-3


@pytest.mark.parametrize("a_mn,b_mn", [(False, False), (False, True), (True, True)])
@pytest.mark.parametrize("M,N,K", [(4096, 2304, 768), (4104, 2000, 520), (8192, 1024, 256)])
def test_gemm_persistent_path(F, a_mn, b_mn, M, N, K):
    """>= one wave of output tiles: persistent CTAs, the TMA producer runs ahead across tile boundaries."""
    torch.manual_seed(M + N)
    dev = _dev()
    A = torch.randn(M, K, device=dev).to(BF16)
    B = torch.randn(N, K, device=dev).to(BF16)
    a = A.t().contiguous() if a_mn else A
    b = B.t().contiguous() if b_mn else B
    bias = torch.randn(N, device=dev)
    ref = A.float() @ B.float().t()
    out = F.gemm(a, b, a_mn=a_mn, b_mn=b_mn, out_dtype=torch.float32)
    assert _rel(out, ref) < 2e-3, _rel(out, ref)
    out2 = F.gemm(a, b, a_mn=a_mn, b_mn=b_mn, bias=bias, act=1)
    assert _rel(out2, torch.relu(ref + bias)) < 1e-2
    acc = torch.ones(M, N, device=dev)
    F.gemm(a, b, a_mn=a_mn, b_mn=b_mn, out=acc, accumulate=True, split_k=1)
    assert _rel(acc, ref + 1.0) < 2e-3


@pytest.mark.parametrize("a_mn,b_mn", [(False, False), (True, True)])
def test_gemm_two_cta_pairs(F, a_mn, b_mn):
    """Deep-K, multi-wave problem with a ragged N tile (a shape the CTA-pair kernel of the Blackwell build served;
    on Hopper it runs on the persistent kernel)."""
    torch.manual_seed(5)
    dev = _dev()
    M, N, K = 4096, 2560 - 8, 2048 + 64          # ragged N tile, K not a multiple of the stage count
    A = torch.randn(M, K, device=dev).to(BF16)
    B = torch.randn(N, K, device=dev).to(BF16)
    a = A.t().contiguous() if a_mn else A
    b = B.t().contiguous() if b_mn else B
    bias = torch.randn(N, device=dev)
    ref = A.float() @ B.float().t()
    out = F.gemm(a, b, a_mn=a_mn, b_mn=b_mn, out_dtype=torch.float32)
    assert _rel(out, ref) < 2e-3, _rel(out, ref)
    out2 = F.gemm(a, b, a_mn=a_mn, b_mn=b_mn, bias=bias, act=1)
    assert _rel(out2, torch.relu(ref + bias)) < 1e-2


@pytest.mark.parametrize("M,N,K", [(8192, 64, 576), (32768, 64, 152), (1000, 72, 64), (32768, 256, 64), (32768, 128, 128),
                                   (20000, 256, 192), (2048, 128, 1152), (512, 256, 2304), (500, 200, 4608)])
def test_gemm_fused_column_statistics(F, M, N, K):
    """BatchNorm statistics taken in the GEMM epilogue (fixed, persistent, CTA-pair and cluster split-K kernels):
    column sums and sums of squares of the bf16 output, ragged M / N included."""
    torch.manual_seed(M + N + K)
    dev = _dev()
    A = torch.randn(M, K, device=dev).to(BF16)
    B = (torch.randn(N, K, device=dev) * 0.2).to(BF16)
    assert F.gemm_stats_fusable(M, N, K)
    stats = torch.zeros(2 * N, device=dev)
    out = F.gemm(A, B, col_stats=stats)
    ref = F.gemm(A, B)
    assert torch.equal(out, ref)
    o = out.float()
    assert _rel(stats[:N], o.sum(0)) < 2e-3, _rel(stats[:N], o.sum(0))
    assert _rel(stats[N:], (o * o).sum(0)) < 2e-3
    F.gemm(A, B, col_stats=stats)                        # accumulates
    assert _rel(stats[N:], 2 * (o * o).sum(0)) < 2e-3


def test_conv_bn_fused_statistics_match_separate_pass(bnn):
    torch.manual_seed(3)
    dev = _dev()
    x = torch.randn(128, 8, 8, 64, device=dev).to(BF16)
    outs = []
    for fused in (False, True):
        torch.manual_seed(4)
        conv = bnn.Conv2d(64, 64, 3, 1, 1).to(dev)
        bn = bnn.BatchNorm2d(64, relu=True).to(dev)
        bn.workspace = torch.zeros(4 * 64, device=dev)
        if fused:
            conv.bn_ws = bn.workspace
        h = conv(x)
        assert (getattr(h, "_bn_stats_ws", None) is not None) == fused
        y = bn(h)
        y.float().sum().backward()
        outs.append((y.detach().clone(), bn.running_mean.clone(), bn.running_var.clone(), bn.workspace[:128].clone(),
                     conv.weight.grad.clone()))
    (y0, m0, v0, s0, g0), (y1, m1, v1, s1, g1) = outs
    assert _rel(s1, s0) < 1e-3
    assert _rel(y1, y0) < 1e-2 and torch.allclose(m0, m1, atol=1e-4) and torch.allclose(v0, v1, rtol=1e-3, atol=1e-4)
    assert _rel(g1, g0) < 2e-2


@pytest.mark.parametrize("c,k,stride,pad,h", [(64, 3, 1, 1, 8), (128, 3, 2, 1, 8), (64, 1, 2, 0, 8), (256, 3, 1, 1, 2)])
def test_tma_im2col_probe_matches_explicit_im2col(F, c, k, stride, pad, h):
    from baton_b200.ops import load
    torch.manual_seed(c + k)
    dev = _dev()
    x = torch.randn(32, h, h, c, device=dev).to(BF16)
    ref, ho, wo, kp = F.im2col(x, k, k, stride, pad)
    assert kp == k * k * c
    col = torch.zeros_like(ref)
    assert load().im2col_tma_probe(x, col, k, k, stride, pad, ho, wo)
    torch.cuda.synchronize()
    assert torch.equal(col, ref)


@pytest.mark.parametrize("cin,cout,k,stride,pad,h,n", [(64, 64, 3, 1, 1, 8, 128), (64, 128, 3, 2, 1, 8, 128),
                                                       (128, 128, 3, 1, 1, 4, 128), (256, 256, 3, 1, 1, 2, 128),
                                                       (64, 128, 1, 2, 0, 8, 128), (64, 64, 3, 1, 1, 5, 7)])
def test_implicit_gemm_conv_matches_im2col_path(F, bnn, cin, cout, k, stride, pad, h, n):
    torch.manual_seed(cin + cout + k)
    dev = _dev()
    x = torch.randn(n, h, h, cin, device=dev).to(BF16)
    torch.manual_seed(1)
    conv = bnn.Conv2d(cin, cout, k, stride, pad).to(dev)
    xi = x.clone().requires_grad_(True)
    y = conv(xi)
    dy = torch.ones_like(y) * 0.5
    y.backward(dy)
    # reference: the explicit im2col / col2im + GEMM lowering the layer takes for shapes implicit GEMM declines
    w2d = conv._w_bf16()
    col, ho, wo, _ = F.im2col(x, k, k, stride, pad)
    dy2 = dy.reshape(n * ho * wo, cout)
    y_ref = F.gemm(col, w2d).view(n, ho, wo, cout)
    dx_ref = F.col2im(F.gemm(dy2, w2d, b_mn=True), (n, h, h, cin), k, k, stride, pad, ho, wo)
    dw_ref = F.gemm(dy2, col, a_mn=True, b_mn=True, out_dtype=torch.float32, accumulate=True)
    dw_ref = dw_ref.view(cout, k, k, cin).permute(0, 3, 1, 2)
    assert _rel(y.detach(), y_ref) < 1e-2
    assert _rel(xi.grad, dx_ref) < 1e-2
    assert _rel(conv.weight.grad, dw_ref) < 1e-2


def test_gemm_simt_fallback_small_pitch(F):
    torch.manual_seed(2)
    dev = _dev()
    M, N, K = 256, 10, 512
    A = torch.randn(M, K, device=dev).to(BF16)
    W = torch.randn(N, K, device=dev).to(BF16)
    dy = torch.randn(M, N, device=dev).to(BF16)       # pitch 10 -> not TMA-able
    dx = F.gemm(dy, W, b_mn=True)
    assert _rel(dx, dy.float() @ W.float()) < 1e-2
    dw = F.gemm(dy, A, a_mn=True, b_mn=True, out_dtype=torch.float32, accumulate=True)
    assert _rel(dw, dy.float().t() @ A.float()) < 2e-3
    y = F.gemm(A, W, out_dtype=torch.float32)          # tiny N through TMA with OOB rows
    assert _rel(y, A.float() @ W.float().t()) < 2e-3


# ------------------------------------------------------------------ optimizer / elementwise
@pytest.mark.parametrize("momentum,nesterov,wd", [(0.0, False, 0.0), (0.9, False, 5e-4), (0.9, True, 1e-4)])
def test_fused_sgd_matches_torch(F, momentum, nesterov, wd):
    torch.manual_seed(3)
    dev = _dev()
    n = 1_000_004
    w = torch.randn(n, device=dev)
    ref_p = torch.nn.Parameter(w.clone())
    opt = torch.optim.SGD([ref_p], lr=0.1, momentum=momentum, nesterov=nesterov, weight_decay=wd)
    g_all = [torch.randn(n, device=dev) for _ in range(3)]
    mom = torch.zeros(n, device=dev) if momentum else None
    wb = torch.zeros(n, device=dev, dtype=BF16)
    hyper = torch.tensor([0.1, momentum, wd, 0.0], device=dev)
    for g in g_all:
        ref_p.grad = g.clone()
        opt.step()
        gg = g.clone()
        F.fused_sgd(w, gg, hyper, mom, wb, zero_grad=True, nesterov=nesterov)
        assert float(gg.abs().max()) == 0.0
    assert torch.allclose(w, ref_p.detach(), atol=1e-5, rtol=1e-5)
    assert torch.equal(wb, w.to(BF16))


def test_weighted_sum_cast_gather_colsum(F):
    torch.manual_seed(4)
    dev = _dev()
    srcs = [torch.randn(100_003, device=dev) for _ in range(5)]
    ws = [0.1, 0.2, 0.3, 0.15, 0.25]
    dst = torch.empty(100_003, device=dev)
    F.weighted_sum_(dst, srcs, ws)
    assert torch.allclose(dst, sum(w * s for w, s in zip(ws, srcs)), atol=1e-5)
    s16 = [s.to(BF16) for s in srcs]
    d16 = torch.empty(100_003, device=dev, dtype=BF16)
    F.weighted_sum_(d16, s16, ws)
    assert _rel(d16, sum(w * s.float() for w, s in zip(ws, s16))) < 1e-2
    x = torch.randn(777, 33, device=dev)
    assert torch.equal(F.cast(x, BF16), x.to(BF16))
    assert torch.equal(F.cast(x.to(BF16), torch.float32), x.to(BF16).float())
    X = torch.randn(500, 32, 32, 8, device=dev).to(BF16)
    idx = torch.randint(0, 500, (64,), device=dev)
    assert torch.equal(F.gather_rows(X, idx), X[idx])
    yl = torch.randint(0, 10, (500,), device=dev)
    assert torch.equal(F.gather_rows(yl, idx), yl[idx])
    m = torch.randn(3000, 70, device=dev).to(BF16)
    out = torch.zeros(70, device=dev)
    F.colsum_(m, out)
    assert _rel(out, m.float().sum(0)) < 1e-3
    for rows, cols in ((3000, 72), (16384, 768), (33, 3072), (5000, 264)):     # 16-byte path, ragged chunks
        m = torch.randn(rows, cols, device=dev).to(BF16)
        out = torch.ones(cols, device=dev)
        F.colsum_(m, out)
        assert _rel(out, m.float().sum(0) + 1.0) < 1e-3, (rows, cols)
    for n in (5000, 4096, 8 * 1000 + 8):                                        # scalar and 16-byte GELU paths
        xv, gv = torch.randn(n, device=dev).to(BF16), torch.randn(n, device=dev).to(BF16)
        xr2 = xv.float().requires_grad_(True)
        yr2 = torch.nn.functional.gelu(xr2, approximate="tanh")
        assert _rel(F.gelu(xv), yr2) < 1e-2
        yr2.backward(gv.float())
        assert _rel(F.gelu_bwd(xv, gv), xr2.grad) < 2e-2
    a, b = torch.randn(4096, device=dev).to(BF16), torch.randn(4096, device=dev).to(BF16)
    assert torch.equal(F.add(a, b, relu=True), torch.relu(a.float() + b.float()).to(BF16))
    assert torch.equal(F.relu_bwd(a, b), torch.where(a > 0, b, torch.zeros_like(b)))
    xg = torch.randn(5000, device=dev).to(BF16)
    assert _rel(F.gelu(xg), torch.nn.functional.gelu(xg.float(), approximate="tanh")) < 1e-2
    xr = xg.float().requires_grad_(True)
    torch.nn.functional.gelu(xr, approximate="tanh").backward(b[:1].float().expand(5000).clone())
    assert _rel(F.gelu_bwd(xg, b[:1].expand(5000).contiguous()), xr.grad) < 2e-2


# ------------------------------------------------------------------ conv plumbing
@pytest.mark.parametrize("cin,k,stride,pad,h", [(64, 3, 1, 1, 8), (64, 3, 2, 1, 8), (3, 7, 2, 3, 32), (64, 1, 2, 0, 8),
                                                (512, 3, 1, 1, 1), (256, 3, 2, 1, 1)])
def test_conv2d_forward_backward_vs_torch(bnn, cin, k, stride, pad, h):
    torch.manual_seed(5)
    dev = _dev()
    n, cout = 16, 128
    conv = bnn.Conv2d(cin, cout, k, stride, pad).to(dev)
    x = torch.randn(n, h, h, cin, device=dev).to(BF16).requires_grad_(cin != 3)
    y = conv(x)
    w32 = conv.weight.detach().to(BF16).float().contiguous().requires_grad_(True)
    x32 = x.detach().float().permute(0, 3, 1, 2).requires_grad_(True)
    yr = torch.nn.functional.conv2d(x32, w32, None, stride, pad)
    assert y.shape == yr.permute(0, 2, 3, 1).shape
    assert _rel(y, yr.permute(0, 2, 3, 1)) < 1e-2
    dy = torch.randn_like(y)
    y.backward(dy)
    yr.backward(dy.float().permute(0, 3, 1, 2))
    assert _rel(conv.weight.grad, w32.grad) < 1e-2
    if cin != 3:
        assert _rel(x.grad, x32.grad.permute(0, 2, 3, 1)) < 1.5e-2


def test_maxpool_avgpool(bnn):
    torch.manual_seed(6)
    dev = _dev()
    x = torch.randn(8, 16, 16, 64, device=dev).to(BF16).requires_grad_(True)
    y = bnn.MaxPool2d(3, 2, 1)(x)
    x32 = x.detach().float().permute(0, 3, 1, 2).requires_grad_(True)
    yr = torch.nn.functional.max_pool2d(x32, 3, 2, 1)
    assert torch.equal(y.float(), yr.permute(0, 2, 3, 1))
    dy = torch.randn_like(y)
    y.backward(dy)
    yr.backward(dy.float().permute(0, 3, 1, 2))
    assert _rel(x.grad, x32.grad.permute(0, 2, 3, 1)) < 1e-2
    x2 = torch.randn(8, 4, 4, 64, device=dev).to(BF16).requires_grad_(True)
    y2 = bnn.GlobalAvgPool()(x2)
    assert _rel(y2, x2.float().mean((1, 2))) < 1e-2
    y2.backward(torch.ones_like(y2))
    assert _rel(x2.grad, torch.full_like(x2, 1 / 16).float()) < 1e-2


# ------------------------------------------------------------------ normalisation
@pytest.mark.parametrize("n,h,c", [(32, 8, 64), (128, 8, 64), (9, 5, 128), (128, 1, 512), (7, 3, 24), (3, 2, 2048)])
@pytest.mark.parametrize("relu,with_res", [(False, False), (True, False), (True, True)])
def test_batchnorm_fwd_bwd(bnn, relu, with_res, n, h, c):
    """Channel counts cover the vectorised column reductions (C/8 a power of two), ragged row counts, and the
    scalar fallback (24 channels); 2048 channels = one thread group per row."""
    torch.manual_seed(7)
    dev = _dev()
    bn = bnn.BatchNorm2d(c, relu=relu).to(dev)
    with torch.no_grad():
        bn.weight.uniform_(0.5, 1.5)
        bn.bias.uniform_(-0.5, 0.5)
    ref = torch.nn.BatchNorm2d(c).to(dev)
    ref.load_state_dict(bn.state_dict())
    x = (torch.randn(n, h, h, c, device=dev) * 2 + 0.5).to(BF16).requires_grad_(True)
    res = torch.randn(n, h, h, c, device=dev).to(BF16).requires_grad_(True) if with_res else None
    y = bn(x, res)
    x32 = x.detach().float().permute(0, 3, 1, 2).requires_grad_(True)
    yr = ref(x32)
    r32 = None
    if with_res:
        r32 = res.detach().float().permute(0, 3, 1, 2).requires_grad_(True)
        yr = yr + r32
    pre_act = yr.detach()
    if relu:
        yr = torch.relu(yr)
    assert _rel(y, yr.permute(0, 2, 3, 1)) < 1.5e-2
    assert torch.allclose(bn.running_mean, ref.running_mean, atol=2e-3)
    assert torch.allclose(bn.running_var, ref.running_var, atol=2e-2, rtol=2e-2)
    assert int(bn.num_batches_tracked) == 1
    dy = torch.randn_like(y)
    y.backward(dy)
    yr.backward(dy.float().permute(0, 3, 1, 2))
    # an output within rounding distance of the ReLU kink may land on the other side of it (bf16 output, fp32
    # atomics in the statistics): such an element's gradient is legitimately dy instead of 0 -- compare away
    # from the kink
    pre = pre_act.permute(0, 2, 3, 1)
    clear = (pre.abs() > 2e-2).float() if relu else torch.ones_like(pre)
    assert _rel(x.grad.float() * clear, x32.grad.permute(0, 2, 3, 1) * clear) < 3e-2
    assert _rel(bn.weight.grad, ref.weight.grad) < 3e-2
    assert _rel(bn.bias.grad, ref.bias.grad) < 3e-2
    if with_res:
        assert _rel(res.grad.float() * clear, r32.grad.permute(0, 2, 3, 1) * clear) < 1e-2


@pytest.mark.parametrize("n,h,c,relu,two", [(128, 8, 64, True, True), (128, 8, 64, False, False), (128, 4, 128, True, True),
                                            (128, 2, 256, True, False), (128, 1, 512, True, True), (9, 5, 128, True, True),
                                            (128, 16, 64, True, False), (32, 8, 256, True, True)])
def test_batchnorm_backward_cluster_kernel_matches_two_kernel_path(bnn, n, h, c, relu, two):
    """Single-kernel BatchNorm backward (one thread-block cluster per 16-channel slice, csrc/norm.cu) against the
    reduce + apply pair, including the two-piece gradient (dy = dy_a + dy_b) and every register-cache depth."""
    from baton_b200.ops import load
    C_ = load()
    torch.manual_seed(13)
    dev = _dev()
    rows = n * h * h
    x = (torch.randn(rows, c, device=dev) * 2 + 0.5).to(BF16)
    mean = x.float().mean(0)
    rstd = (x.float().var(0, unbiased=False) + 1e-5).rsqrt()
    gamma = torch.rand(c, device=dev) + 0.5
    y = (torch.randn(rows, c, device=dev)).to(BF16)            # only its sign matters (ReLU mask)
    dy_a = torch.randn(rows, c, device=dev).to(BF16)
    dy_b = torch.randn(rows, c, device=dev).to(BF16) if two else None
    dy = dy_a if dy_b is None else (dy_a.float() + dy_b.float())
    # fp32 oracle
    g = dy.float() * ((y.float() > 0).float() if relu else 1.0)
    xh = (x.float() - mean) * rstd
    dxr = gamma * rstd * (g - g.mean(0) - xh * (g * xh).mean(0))
    dgr, dbr = (g * xh).sum(0), g.sum(0)
    dx = torch.empty_like(x)
    dres = torch.empty_like(x)
    dg = torch.ones(c, device=dev)       # accumulate semantics: starts at 1
    db = torch.ones(c, device=dev)
    for cap in (16, 8, 2, -2):          # negative: allow the uncached (re-reading) variant for row counts beyond the cache
        dg.fill_(1.0); db.fill_(1.0)
        ok = C_.bn_bwd_cluster(x, y, dy_a, dy_b, dx, dres, gamma, mean, rstd, dg, db, rows, c, relu, cap)
        torch.cuda.synchronize()
        if not ok:
            assert cap > 0 and rows > cap * 1024
            continue
        assert _rel(dx, dxr) < 2e-2
        assert _rel(dres, g) < 1e-2
        assert _rel(dg - 1.0, dgr) < 1e-2 and _rel(db - 1.0, dbr) < 1e-2


@pytest.mark.parametrize("n,h,c,two", [(128, 16, 64, True), (8, 16, 64, False), (5, 9, 32, True), (16, 7, 128, True)])
def test_stem_bn_relu_maxpool_fused_matches_separate_kernels(F, n, h, c, two):
    """ResNet stem: BatchNorm + ReLU + 3x3/2 max-pool in one kernel (the normalised activation is never written) must be
    BIT-identical to bn_apply + maxpool, and its backward (BatchNorm sums over the pooled gradient, gather in the apply
    pass) must match maxpool_bwd + BatchNorm backward and an fp32 autograd oracle."""
    from baton_b200.ops import load
    C_ = load()
    torch.manual_seed(3 + n + h)
    dev = _dev()
    k, stride, pad = 3, 2, 1
    rows = n * h * h
    z = (torch.randn(n, h, h, c, device=dev) * 1.5 + 0.3).to(BF16)
    sums = torch.cat([z.float().sum((0, 1, 2)), (z.float() ** 2).sum((0, 1, 2))]).contiguous()
    gamma = torch.rand(c, device=dev) + 0.5
    beta = torch.randn(c, device=dev) * 0.3
    rm, rv = torch.zeros(c, device=dev), torch.ones(c, device=dev)
    rm2, rv2 = rm.clone(), rv.clone()
    nbt, nbt2 = torch.zeros((), dtype=torch.long, device=dev), torch.zeros((), dtype=torch.long, device=dev)
    # separate kernels
    y = torch.empty_like(z)
    mean, rstd = torch.empty(c, device=dev), torch.empty(c, device=dev)
    C_.bn_apply(z, None, y, sums, gamma, beta, rm, rv, mean, rstd, nbt, rows, c, 1e-5, 0.1, True, True)
    p_ref, arg_ref = F.maxpool(y, k, stride, pad)
    out = F.bn_relu_maxpool(z, sums, gamma, beta, rm2, rv2, nbt2, 1e-5, 0.1, k, stride, pad)
    assert out is not None
    p, arg, mean2, rstd2 = out
    torch.cuda.synchronize()
    assert torch.equal(p, p_ref) and torch.equal(arg, arg_ref)
    assert torch.equal(mean, mean2) and torch.equal(rstd, rstd2)
    assert torch.equal(rm, rm2) and torch.equal(rv, rv2) and int(nbt2) == 1
    # backward
    dy_a = torch.randn_like(p)
    dy_b = torch.randn_like(p) if two else None
    dyd = F.maxpool_bwd(dy_a, arg_ref, tuple(z.shape), k, stride, pad, dy_b=dy_b)
    sb = torch.zeros(2 * c, device=dev)
    dz_ref, dg_ref, db_ref = torch.empty_like(z), torch.ones(c, device=dev), torch.ones(c, device=dev)
    C_.bn_bwd_reduce(z, y, dyd, mean, rstd, sb, rows, c, True)
    C_.bn_bwd_apply(z, y, dyd, dz_ref, None, gamma, mean, rstd, sb, dg_ref, db_ref, rows, c, True)
    sb2 = torch.zeros(2 * c, device=dev)
    dg, db = torch.ones(c, device=dev), torch.ones(c, device=dev)
    dz = F.bn_maxpool_bwd(z, p, arg, dy_a, dy_b, gamma, mean2, rstd2, sb2, dg, db, k, stride, pad)
    torch.cuda.synchronize()
    assert dz is not None
    assert _rel(sb2, sb) < 1e-2            # the separate path rounds the scattered gradient to bf16 first
    assert _rel(dz, dz_ref) < 1e-2
    assert _rel(dg - 1.0, dg_ref - 1.0) < 5e-3 and _rel(db - 1.0, db_ref - 1.0) < 5e-3
    # fp32 autograd oracle of the whole stem tail
    z32 = z.float().requires_grad_(True)
    g32, b32 = gamma.clone().requires_grad_(True), beta.clone().requires_grad_(True)
    zn = z32.permute(0, 3, 1, 2)
    yn = torch.relu(torch.nn.functional.batch_norm(zn, None, None, g32, b32, True, 0.1, 1e-5))
    # the kernels pick the window maximum among bf16-rounded candidates: round with a straight-through estimator so the
    # oracle routes the gradient to the same positions (exact bf16 ties may still go to another tap: compare dz by
    # direction and by the fraction of elements that differ, not by the worst element)
    yq = yn + (yn.to(BF16).float() - yn).detach()
    pn = torch.nn.functional.max_pool2d(yq, k, stride, pad)
    dyt = dy_a.float() + (dy_b.float() if dy_b is not None else 0.0)
    pn.backward(dyt.permute(0, 3, 1, 2))
    assert _rel(p, pn.permute(0, 2, 3, 1)) < 1e-2
    ref = z32.grad
    cos = torch.nn.functional.cosine_similarity(dz.float().flatten(), ref.flatten(), dim=0)
    assert float(cos) > 0.99, float(cos)
    bad = ((dz.float() - ref).abs() > 0.05 * ref.abs().max()).float().mean()
    assert float(bad) < 0.01, float(bad)
    assert _rel(dg - 1.0, g32.grad) < 3e-2 and _rel(db - 1.0, b32.grad) < 3e-2


def test_layernorm_softmax(bnn):
    torch.manual_seed(8)
    dev = _dev()
    rows, c = 512, 768
    ln = bnn.LayerNorm(c, eps=1e-12).to(dev)
    with torch.no_grad():
        ln.weight.uniform_(0.5, 1.5)
        ln.bias.uniform_(-0.5, 0.5)
    x = torch.randn(rows, c, device=dev).to(BF16).requires_grad_(True)
    r = torch.randn(rows, c, device=dev).to(BF16).requires_grad_(True)
    y = ln(x, r)
    x32 = x.detach().float().requires_grad_(True)
    r32 = r.detach().float().requires_grad_(True)
    w32, b32 = ln.weight.detach().clone().requires_grad_(True), ln.bias.detach().clone().requires_grad_(True)
    yr = torch.nn.functional.layer_norm((x32 + r32).to(BF16).float(), (c,), w32, b32, 1e-12)
    assert _rel(y, yr) < 1.5e-2
    dy = torch.randn_like(y)
    y.backward(dy)
    yr.backward(dy.float())
    assert _rel(ln.weight.grad, w32.grad) < 3e-2 and _rel(ln.bias.grad, b32.grad) < 3e-2
    s = torch.randn(64, 12, 128, 128, device=dev).to(BF16).requires_grad_(True)
    p = bnn.softmax(s, 0.125)
    s32 = s.detach().float().requires_grad_(True)
    pr = torch.softmax(s32 * 0.125, -1)
    assert _rel(p, pr) < 1e-2
    g = torch.randn_like(p)
    p.backward(g)
    pr.backward(g.float())
    assert _rel(s.grad, s32.grad) < 3e-2


@pytest.mark.parametrize("rows,c", [(37, 64), (101, 128), (77, 256), (65, 512), (33, 1024), (50, 100), (4099, 768)])
def test_row_kernels_all_group_shapes(bnn, rows, c):
    """LayerNorm / softmax row kernels: every (lanes-per-row, vectors-per-lane) instantiation, ragged row counts,
    and the scalar fallback for rows that are not a multiple of 8 elements."""
    torch.manual_seed(rows + c)
    dev = _dev()
    ln = bnn.LayerNorm(c, eps=1e-5).to(dev)
    with torch.no_grad():
        ln.weight.uniform_(0.5, 1.5)
        ln.bias.uniform_(-0.5, 0.5)
    x = torch.randn(rows, c, device=dev).to(BF16).requires_grad_(True)
    y = ln(x)
    x32 = x.detach().float().requires_grad_(True)
    w32, b32 = ln.weight.detach().clone().requires_grad_(True), ln.bias.detach().clone().requires_grad_(True)
    yr = torch.nn.functional.layer_norm(x32, (c,), w32, b32, 1e-5)
    assert _rel(y, yr) < 1.5e-2
    dy = torch.randn_like(y)
    y.backward(dy)
    yr.backward(dy.float())
    assert _rel(x.grad, x32.grad) < 3e-2
    assert _rel(ln.weight.grad, w32.grad) < 3e-2 and _rel(ln.bias.grad, b32.grad) < 3e-2
    s = (torch.randn(rows, c, device=dev) * 2).to(BF16).requires_grad_(True)
    p = bnn.softmax(s, 0.5)
    s32 = s.detach().float().requires_grad_(True)
    pr = torch.softmax(s32 * 0.5, -1)
    assert _rel(p, pr) < 1e-2
    g = torch.randn_like(p)
    p.backward(g)
    pr.backward(g.float())
    assert _rel(s.grad, s32.grad) < 3e-2


# ------------------------------------------------------------------ losses
def test_softmax_xent_and_mse(F, bnn):
    torch.manual_seed(9)
    dev = _dev()
    logits = (torch.randn(256, 10, device=dev) * 3).requires_grad_(True)
    tgt = torch.randint(0, 10, (256,), device=dev)
    loss, stats = bnn.cross_entropy(logits, tgt)
    l32 = logits.detach().clone().requires_grad_(True)
    ref = torch.nn.functional.cross_entropy(l32, tgt)
    assert abs(float(loss) - float(ref)) < 1e-4
    assert int(stats[1]) == int((l32.argmax(-1) == tgt).sum())
    loss.backward()
    ref.backward()
    assert torch.allclose(logits.grad, l32.grad, atol=1e-6)
    lb = (torch.randn(128, 1000, device=dev) * 2).to(BF16)
    tb = torch.randint(0, 1000, (128,), device=dev)
    acc, dl = F.softmax_xent(lb, tb)
    assert abs(float(acc[0]) - float(torch.nn.functional.cross_entropy(lb.float(), tb))) < 2e-3
    p = torch.randn(300, 1, device=dev).requires_grad_(True)
    t = torch.randn(300, 1, device=dev)
    l = bnn.mse_loss(p, t)
    p32 = p.detach().clone().requires_grad_(True)
    lr = torch.nn.functional.mse_loss(p32, t)
    assert abs(float(l) - float(lr)) < 1e-5
    l.backward()
    lr.backward()
    assert torch.allclose(p.grad, p32.grad, atol=1e-6)


@pytest.mark.parametrize("rows,K,nc", [(128, 512, 10), (37, 256, 2), (128, 2048, 32), (5, 64, 1), (200, 72, 7)])
def test_linear_xent_head_one_launch_matches_fp32_reference(F, rows, K, nc):
    """Classifier head (linear + softmax cross-entropy forward AND backward) in one launch vs plain fp32 PyTorch."""
    torch.manual_seed(rows + K + nc)
    dev = _dev()
    x = torch.randn(rows, K, device=dev).to(BF16)
    w = (torch.randn(nc, K, device=dev) * 0.05).to(BF16)
    b = torch.randn(nc, device=dev) * 0.1
    t = torch.randint(0, nc, (rows,), device=dev)
    dw = torch.ones(nc, K, device=dev)                 # accumulate semantics
    db = torch.ones(nc, device=dev)
    acc = torch.zeros(2, device=dev)
    out = F.linear_xent_head(x, w, b, t, dw, db, acc=acc, want_logits=True)
    assert out is not None
    _, dx, logits = out
    torch.cuda.synchronize()
    x32 = x.float().requires_grad_(True)
    w32 = w.float().requires_grad_(True)
    b32 = b.clone().requires_grad_(True)
    ref_logits = x32 @ w32.t() + b32
    loss = torch.nn.functional.cross_entropy(ref_logits, t)
    loss.backward()
    assert _rel(logits, ref_logits) < 1e-4
    assert abs(float(acc[0]) - float(loss)) < 1e-4 * max(1.0, abs(float(loss)))
    assert int(acc[1]) == int((ref_logits.argmax(-1) == t).sum())
    assert _rel(dx, x32.grad) < 1e-2                       # bf16 output
    assert _rel(dw - 1.0, w32.grad) < 1e-4 and _rel(db - 1.0, b32.grad) < 1e-4
