"""Halo-tiled 3x3 stride-1 convolution (csrc/conv_halo.cu) against the im2col-mode implicit GEMM and fp32 torch."""
import pytest
import torch

from baton_b200.ops import functional as F

pytestmark = pytest.mark.gpu
BF16 = torch.bfloat16

# (batch, cluster size) on 8x8 maps, one image per 64-row tile: full clusters of 4 and 2, a batch whose tile count only
# a cluster of 2 divides (126), odd tile counts (3, 1); partial last tiles are in test_other_image_sizes
CASES = [(128, 4), (128, 2), (128, 1), (126, 2), (126, 1), (3, 1), (1, 1)]


def _data(n, h=8, cin=64, cout=64, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(n, h, h, cin, device="cuda", generator=g).to(BF16)
    w2d = (torch.randn(cout, 9 * cin, device="cuda", generator=g) * 0.05).to(BF16)
    return x, w2d


def _w4(w2d, cin):   # channels_last [Cout, 9*Cin] -> OIHW fp32
    return w2d.float().view(w2d.shape[0], 3, 3, cin).permute(0, 3, 1, 2)


def _close(got, ref, tol=2e-2):
    err = (got.float() - ref).abs().max().item()
    assert err <= tol * max(ref.abs().max().item(), 1.0), err


@pytest.mark.parametrize("n,mc", CASES)
def test_forward_matches_im2col_path_and_torch(n, mc):
    x, w2d = _data(n)
    y_old = F.conv_igemm_fwd(x, w2d, 3, 3, 1, 1, path="im2col")
    y = F.conv_igemm_fwd(x, w2d, 3, 3, 1, 1, path="halo", mc=mc)
    torch.cuda.synchronize()
    # same k order (tap-major, then 4 x k16 over the 64 channels), one channel block: the same bits
    assert torch.equal(y, y_old)
    ref = torch.nn.functional.conv2d(x.float().permute(0, 3, 1, 2), _w4(w2d, 64), padding=1)
    _close(y, ref.permute(0, 2, 3, 1).reshape(-1, 64))


@pytest.mark.parametrize("n,mc", CASES)
@pytest.mark.parametrize("cin", [64, 128])
def test_dgrad_matches_im2col_path_and_torch(n, mc, cin):
    dy, _ = _data(n, seed=1)
    _, w2d = _data(1, cin=cin, cout=64, seed=2)
    dx_old = F.conv_igemm_dgrad(dy, w2d, (n, 8, 8, cin), 3, 3, 1, path="im2col")
    dx = F.conv_igemm_dgrad(dy, w2d, (n, 8, 8, cin), 3, 3, 1, path="halo", mc=mc)
    torch.cuda.synchronize()
    assert torch.equal(dx, dx_old)
    ref = torch.nn.grad.conv2d_input((n, cin, 8, 8), _w4(w2d, cin), dy.float().permute(0, 3, 1, 2), padding=1)
    _close(dx, ref.permute(0, 2, 3, 1))


@pytest.mark.parametrize("n,mc", CASES)
def test_fused_column_statistics(n, mc):
    x, w2d = _data(n, seed=3)
    stats = torch.zeros(128, device="cuda")
    y = F.conv_igemm_fwd(x, w2d, 3, 3, 1, 1, col_stats=stats, path="halo", mc=mc)
    torch.cuda.synchronize()
    yf = y.float()
    torch.testing.assert_close(stats[:64], yf.sum(0), rtol=1e-4, atol=1e-2)
    torch.testing.assert_close(stats[64:], (yf * yf).sum(0), rtol=1e-4, atol=1e-2)


# several images per 64-row tile; 6 and 3 images of 4x4 leave a partial last tile (rows past M, zero-filled halo)
@pytest.mark.parametrize("n,h,w,mc", [(16, 4, 4, 4), (6, 4, 4, 2), (3, 4, 4, 1), (16, 2, 2, 1), (16, 4, 8, 2)])
def test_other_image_sizes(n, h, w, mc):
    g = torch.Generator(device="cuda").manual_seed(4)
    x = torch.randn(n, h, w, 64, device="cuda", generator=g).to(BF16)
    w2d = (torch.randn(64, 576, device="cuda", generator=g) * 0.05).to(BF16)
    assert F.halo_eligible(3, 3, 1, 1, 64, h, w)
    stats = torch.zeros(128, device="cuda")
    y = F.conv_igemm_fwd(x, w2d, 3, 3, 1, 1, col_stats=stats, path="halo", mc=mc)
    y_old = F.conv_igemm_fwd(x, w2d, 3, 3, 1, 1, path="im2col")
    dx = F.conv_igemm_dgrad(x, w2d, (n, h, w, 64), 3, 3, 1, path="halo", mc=mc)
    dx_old = F.conv_igemm_dgrad(x, w2d, (n, h, w, 64), 3, 3, 1, path="im2col")
    torch.cuda.synchronize()
    assert torch.equal(y, y_old) and torch.equal(dx, dx_old)
    torch.testing.assert_close(stats[:64], y.float().sum(0), rtol=1e-4, atol=1e-2)


def test_graph_captured_layer1_chain_matches_eager():
    """Two layer1 convolutions forward and their two input gradients, captured into one graph (PDL edges, clusters)."""
    x, w1 = _data(128, seed=5)
    _, w2 = _data(1, seed=6)
    dy, _ = _data(128, seed=7)
    stats = torch.zeros(2, 128, device="cuda")

    def chain():
        stats.zero_()
        a = F.conv_igemm_fwd(x, w1, 3, 3, 1, 1, col_stats=stats[0])
        b = F.conv_igemm_fwd(a.view(128, 8, 8, 64), w2, 3, 3, 1, 1, col_stats=stats[1])
        da = F.conv_igemm_dgrad(dy, w2, (128, 8, 8, 64), 3, 3, 1)
        dx = F.conv_igemm_dgrad(da, w1, (128, 8, 8, 64), 3, 3, 1)
        return b, dx

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


def test_flagship_step_launches_the_halo_kernel_eight_times(monkeypatch):
    """ResNet-18, 32x32, batch 128: the four layer1 convolutions forward and their four input gradients."""
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

            def counted(*args):
                calls.append(args[3])
                return fn(*args)
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
    assert sorted(calls) == [False] * 4 + [True] * 4
