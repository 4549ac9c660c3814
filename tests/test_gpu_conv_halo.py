"""Halo-tiled 3x3 convolution (csrc/conv_halo.cu, ResNet layer1 and layer2 shapes) against the im2col-mode implicit
GEMM with cluster split-K 1 and against fp32 torch."""
import pytest
import torch

from baton_b200.ops import functional as F

pytestmark = pytest.mark.gpu
BF16 = torch.bfloat16

# (gathered channels, input size, stride) of the three forms at their ResNet-18 shapes: layer1 (64 -> 64, 8x8),
# layer2.0.conv1 (stride 2, 64 -> 128, 8x8 -> 4x4) and the stride-1 layer2 convolutions (128 -> 128, 4x4)
LAYER1, LAYER2_S2, LAYER2 = (64, 8, 1), (64, 8, 2), (128, 4, 1)
# (batch, cluster size).  Layer1: one 8x8 image per 64-row tile: full clusters of 4 and 2, a batch whose tile count
# only a cluster of 2 divides (126), odd tile counts (3, 1); partial last tiles are in test_other_image_sizes.
# Layer2: 4x4 output maps, four images per tile: 128 and 126 (a partial last tile) give 32 tiles, which every cluster
# size divides; 3 and 1 give one tile.
LAYER1_CASES = [(128, 4), (128, 2), (128, 1), (126, 2), (126, 1), (3, 1), (1, 1)]
LAYER2_CASES = [(n, mc) for n in (128, 126) for mc in (1, 2, 4, 8)] + [(3, 1), (1, 1)]
FORWARD_CASES = ([LAYER1 + c for c in LAYER1_CASES] + [LAYER2_S2 + c for c in LAYER2_CASES] +
                 [LAYER2 + c for c in LAYER2_CASES])


def _data(n, h, cin, cout, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(n, h, h, cin, device="cuda", generator=g).to(BF16)
    w2d = (torch.randn(cout, 9 * cin, device="cuda", generator=g) * 0.05).to(BF16)
    return x, w2d


def _w4(w2d, cin):   # channels_last [Cout, 9*Cin] -> OIHW fp32
    return w2d.float().view(w2d.shape[0], 3, 3, cin).permute(0, 3, 1, 2)


def _close(got, ref, tol=2e-2):
    err = (got.float() - ref).abs().max().item()
    assert err <= tol * max(ref.abs().max().item(), 1.0), err


def _cout(cin, stride):   # output channels of the convolution at its ResNet-18 shape
    return 64 if (cin, stride) == (64, 1) else 128


@pytest.mark.parametrize("cin,h,stride,n,mc", FORWARD_CASES)
def test_forward_matches_im2col_path_and_torch(cin, h, stride, n, mc):
    cout = _cout(cin, stride)
    x, w2d = _data(n, h, cin, cout)
    assert F.halo_eligible(3, 3, stride, 1, cin, h, h)
    y_old = F.conv_igemm_fwd(x, w2d, 3, 3, stride, 1, path="im2col", cluster_k=1)
    y = F.conv_igemm_fwd(x, w2d, 3, 3, stride, 1, path="halo", mc=mc)
    torch.cuda.synchronize()
    # same k order (tap-major, then channel block, then 4 x k16), one pass over K: the same bits
    assert torch.equal(y, y_old)
    ref = torch.nn.functional.conv2d(x.float().permute(0, 3, 1, 2), _w4(w2d, cin), stride=stride, padding=1)
    _close(y, ref.permute(0, 2, 3, 1).reshape(-1, cout))


# (gathered channels = Cout, input size, Cin): layer1 with 64 and 128 input channels, the stride-1 layer2 convolutions
@pytest.mark.parametrize("cout,h,cin,n,mc", [(64, 8, cin) + c for cin in (64, 128) for c in LAYER1_CASES] +
                         [(128, 4, 128) + c for c in LAYER2_CASES])
def test_dgrad_matches_im2col_path_and_torch(cout, h, cin, n, mc):
    dy, _ = _data(n, h, cout, cout, seed=1)
    _, w2d = _data(1, h, cin, cout, seed=2)
    dx_old = F.conv_igemm_dgrad(dy, w2d, (n, h, h, cin), 3, 3, 1, path="im2col", cluster_k=1)
    dx = F.conv_igemm_dgrad(dy, w2d, (n, h, h, cin), 3, 3, 1, path="halo", mc=mc)
    torch.cuda.synchronize()
    assert torch.equal(dx, dx_old)
    ref = torch.nn.grad.conv2d_input((n, cin, h, h), _w4(w2d, cin), dy.float().permute(0, 3, 1, 2), padding=1)
    _close(dx, ref.permute(0, 2, 3, 1))


@pytest.mark.parametrize("cin,h,stride,n,mc", [LAYER1 + c for c in LAYER1_CASES] +
                         [f + c for f in (LAYER2_S2, LAYER2) for c in ((128, 4), (126, 8), (3, 1))])
def test_fused_column_statistics(cin, h, stride, n, mc):
    cout = _cout(cin, stride)
    x, w2d = _data(n, h, cin, cout, seed=3)
    stats = torch.zeros(2 * cout, device="cuda")
    y = F.conv_igemm_fwd(x, w2d, 3, 3, stride, 1, col_stats=stats, path="halo", mc=mc)
    torch.cuda.synchronize()
    yf = y.float()
    torch.testing.assert_close(stats[:cout], yf.sum(0), rtol=1e-4, atol=1e-2)
    torch.testing.assert_close(stats[cout:], (yf * yf).sum(0), rtol=1e-4, atol=1e-2)


# several images per 64-row tile (4x4, 2x2, 4x8 over 64 channels; 2x2 over 128; stride 2 onto 2x2 outputs), one 8x8
# image per tile (128 channels; stride 2 onto 8x8 outputs); 6 and 3 images of 4x4 leave a partial last tile (rows past
# M, zero-filled halo)
@pytest.mark.parametrize("n,cin,h,w,stride,mc", [
    (16, 64, 4, 4, 1, 4), (6, 64, 4, 4, 1, 2), (3, 64, 4, 4, 1, 1), (16, 64, 2, 2, 1, 1), (16, 64, 4, 8, 1, 2),
    (32, 128, 2, 2, 1, 2), (4, 128, 8, 8, 1, 4), (6, 128, 4, 4, 1, 2), (32, 64, 4, 4, 2, 2), (4, 64, 16, 16, 2, 4)])
def test_other_image_sizes(n, cin, h, w, stride, mc):
    cout = _cout(cin, stride)
    g = torch.Generator(device="cuda").manual_seed(4)
    x = torch.randn(n, h, w, cin, device="cuda", generator=g).to(BF16)
    w2d = (torch.randn(cout, 9 * cin, device="cuda", generator=g) * 0.05).to(BF16)
    assert F.halo_eligible(3, 3, stride, 1, cin, h, w)
    stats = torch.zeros(2 * cout, device="cuda")
    y = F.conv_igemm_fwd(x, w2d, 3, 3, stride, 1, col_stats=stats, path="halo", mc=mc)
    y_old = F.conv_igemm_fwd(x, w2d, 3, 3, stride, 1, path="im2col", cluster_k=1)
    torch.cuda.synchronize()
    assert torch.equal(y, y_old)
    torch.testing.assert_close(stats[:cout], y.float().sum(0), rtol=1e-4, atol=1e-2)
    if stride == 1:
        dx = F.conv_igemm_dgrad(x, w2d, (n, h, w, cin), 3, 3, 1, path="halo", mc=mc)
        dx_old = F.conv_igemm_dgrad(x, w2d, (n, h, w, cin), 3, 3, 1, path="im2col", cluster_k=1)
        torch.cuda.synchronize()
        assert torch.equal(dx, dx_old)


def _graph_matches_eager(chain, stats):
    eager = [t.clone() for t in chain()]
    eager_stats = stats.clone()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        chain()
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = chain()
    for _ in range(3):
        g.replay()
    torch.cuda.synchronize()
    for a, b in zip(out, eager):
        assert torch.equal(a, b)
    torch.testing.assert_close(stats, eager_stats, rtol=1e-5, atol=1e-3)


def test_graph_captured_layer1_chain_matches_eager():
    """Two layer1 convolutions forward and their two input gradients, captured into one graph (PDL edges, clusters)."""
    x, w1 = _data(128, 8, 64, 64, seed=5)
    _, w2 = _data(1, 8, 64, 64, seed=6)
    dy, _ = _data(128, 8, 64, 64, seed=7)
    stats = torch.zeros(2, 128, device="cuda")

    def chain():
        stats.zero_()
        a = F.conv_igemm_fwd(x, w1, 3, 3, 1, 1, col_stats=stats[0])
        b = F.conv_igemm_fwd(a.view(128, 8, 8, 64), w2, 3, 3, 1, 1, col_stats=stats[1])
        da = F.conv_igemm_dgrad(dy, w2, (128, 8, 8, 64), 3, 3, 1)
        dx = F.conv_igemm_dgrad(da, w1, (128, 8, 8, 64), 3, 3, 1)
        return b, dx

    _graph_matches_eager(chain, stats)


def test_graph_captured_layer2_chain_matches_eager():
    """layer2.0.conv1 and conv2 forward and conv2's input gradient, captured into one graph (PDL edges, clusters)."""
    x, w1 = _data(128, 8, 64, 128, seed=5)
    _, w2 = _data(1, 4, 128, 128, seed=6)
    dy, _ = _data(128, 4, 128, 128, seed=7)
    stats = torch.zeros(2, 256, device="cuda")

    def chain():
        stats.zero_()
        a = F.conv_igemm_fwd(x, w1, 3, 3, 2, 1, col_stats=stats[0])
        b = F.conv_igemm_fwd(a.view(128, 4, 4, 128), w2, 3, 3, 1, 1, col_stats=stats[1])
        da = F.conv_igemm_dgrad(dy, w2, (128, 4, 4, 128), 3, 3, 1)
        return a, b, da

    _graph_matches_eager(chain, stats)


def test_flagship_step_launches_the_halo_kernel_fifteen_times(monkeypatch):
    """ResNet-18, 32x32, batch 128: the four layer1 convolutions forward and their four input gradients, the four
    layer2 3x3 convolutions forward and the input gradients of the three stride-1 ones."""
    from baton_b200.models import resnet18
    from baton_b200.ops import load
    from baton_b200.ops import nn as bnn
    from baton_b200.parallel.arena import ParamArena

    calls = []

    class Counting:
        def __init__(self, inner):
            self.inner = inner

        def __getattr__(self, name):
            fn = getattr(self.inner, name)
            if name != "conv_halo":
                return fn

            def counted(src, w, out, stride, dgrad, mc, col_stats):
                calls.append((src.shape[3], stride, dgrad))
                return fn(src, w, out, stride, dgrad, mc, col_stats)
            return counted

    counting = Counting(load())
    monkeypatch.setattr(F, "load", lambda: counting)
    dev = torch.device("cuda:0")
    torch.manual_seed(0)
    model = resnet18(10)
    ParamArena(model, dev)
    model.build_workspace(dev)
    model.train()
    x = torch.randn(128, 32, 32, 3, device=dev).to(BF16)
    y = torch.randint(0, 10, (128,), device=dev)
    loss, _ = bnn.cross_entropy(model(x), y)
    loss.backward()
    torch.cuda.synchronize()
    # (gathered channels, stride, dgrad)
    assert sorted(calls) == sorted([(64, 1, False)] * 4 + [(64, 1, True)] * 4 + [(128, 1, False)] * 3 +
                                   [(128, 1, True)] * 3 + [(64, 2, False)])
