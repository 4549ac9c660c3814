"""Wide-channel halo kernel (csrc/conv_halo.cu conv_halo_wide_kernel, ResNet layer2 shapes) against the im2col-mode
implicit GEMM with cluster split-K 1 and against fp32 torch."""
import pytest
import torch

from baton_b200.ops import functional as F

pytestmark = pytest.mark.gpu
BF16 = torch.bfloat16

# (batch, cluster size): 4x4 output maps, four images per 64-row tile.  128 and 126 (a partial last tile) give 32
# tiles, which every cluster size divides; 3 and 1 give one tile.
CASES = [(n, mc) for n in (128, 126) for mc in (1, 2, 4, 8)] + [(3, 1), (1, 1)]
# (gathered channels, input size, stride) of the two forwards: layer2.0.conv1 and the stride-1 128 -> 128 convs
FORWARDS = [(64, 8, 2), (128, 4, 1)]


def _data(n, h, cin, cout=128, seed=0):
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
@pytest.mark.parametrize("cin,h,stride", FORWARDS)
def test_forward_matches_im2col_path_and_torch(n, mc, cin, h, stride):
    x, w2d = _data(n, h, cin)
    assert F.halo_wide_eligible(3, 3, stride, 1, cin, h, h)
    y_old = F.conv_igemm_fwd(x, w2d, 3, 3, stride, 1, path="im2col", cluster_k=1)
    y = F.conv_igemm_fwd(x, w2d, 3, 3, stride, 1, path="halo", mc=mc)
    torch.cuda.synchronize()
    # same k order (tap-major, then channel block, then 4 x k16), one pass over K: the same bits
    assert torch.equal(y, y_old)
    ref = torch.nn.functional.conv2d(x.float().permute(0, 3, 1, 2), _w4(w2d, cin), stride=stride, padding=1)
    _close(y, ref.permute(0, 2, 3, 1).reshape(-1, 128))


@pytest.mark.parametrize("n,mc", CASES)
def test_dgrad_matches_im2col_path_and_torch(n, mc):
    dy, _ = _data(n, 4, 128, seed=1)
    _, w2d = _data(1, 4, 128, seed=2)
    dx_old = F.conv_igemm_dgrad(dy, w2d, (n, 4, 4, 128), 3, 3, 1, path="im2col", cluster_k=1)
    dx = F.conv_igemm_dgrad(dy, w2d, (n, 4, 4, 128), 3, 3, 1, path="halo", mc=mc)
    torch.cuda.synchronize()
    assert torch.equal(dx, dx_old)
    ref = torch.nn.grad.conv2d_input((n, 128, 4, 4), _w4(w2d, 128), dy.float().permute(0, 3, 1, 2), padding=1)
    _close(dx, ref.permute(0, 2, 3, 1))


@pytest.mark.parametrize("n,mc", [(128, 4), (126, 8), (3, 1)])
@pytest.mark.parametrize("cin,h,stride", FORWARDS)
def test_fused_column_statistics(n, mc, cin, h, stride):
    x, w2d = _data(n, h, cin, seed=3)
    stats = torch.zeros(256, device="cuda")
    y = F.conv_igemm_fwd(x, w2d, 3, 3, stride, 1, col_stats=stats, path="halo", mc=mc)
    torch.cuda.synchronize()
    yf = y.float()
    torch.testing.assert_close(stats[:128], yf.sum(0), rtol=1e-4, atol=1e-2)
    torch.testing.assert_close(stats[128:], (yf * yf).sum(0), rtol=1e-4, atol=1e-2)


# other image sizes: 16 images of 2x2 per tile, one 8x8 image per tile, and stride 2 onto 2x2 and 8x8 outputs;
# 6 images of 4x4 leave a partial last tile
@pytest.mark.parametrize("n,cin,h,stride,mc", [(32, 128, 2, 1, 2), (4, 128, 8, 1, 4), (6, 128, 4, 1, 2),
                                               (32, 64, 4, 2, 2), (4, 64, 16, 2, 4)])
def test_other_image_sizes(n, cin, h, stride, mc):
    x, w2d = _data(n, h, cin, seed=4)
    assert F.halo_wide_eligible(3, 3, stride, 1, cin, h, h)
    stats = torch.zeros(256, device="cuda")
    y = F.conv_igemm_fwd(x, w2d, 3, 3, stride, 1, col_stats=stats, path="halo", mc=mc)
    y_old = F.conv_igemm_fwd(x, w2d, 3, 3, stride, 1, path="im2col", cluster_k=1)
    torch.cuda.synchronize()
    assert torch.equal(y, y_old)
    torch.testing.assert_close(stats[:128], y.float().sum(0), rtol=1e-4, atol=1e-2)
    if stride == 1:
        dx = F.conv_igemm_dgrad(x, w2d, (n, h, h, 128), 3, 3, 1, path="halo", mc=mc)
        dx_old = F.conv_igemm_dgrad(x, w2d, (n, h, h, 128), 3, 3, 1, path="im2col", cluster_k=1)
        torch.cuda.synchronize()
        assert torch.equal(dx, dx_old)


def test_graph_captured_layer2_chain_matches_eager():
    """layer2.0.conv1 and conv2 forward and conv2's input gradient, captured into one graph (PDL edges, clusters)."""
    x, w1 = _data(128, 8, 64, seed=5)
    _, w2 = _data(1, 4, 128, seed=6)
    dy, _ = _data(128, 4, 128, seed=7)
    stats = torch.zeros(2, 256, device="cuda")

    def chain():
        stats.zero_()
        a = F.conv_igemm_fwd(x, w1, 3, 3, 2, 1, col_stats=stats[0])
        b = F.conv_igemm_fwd(a.view(128, 4, 4, 128), w2, 3, 3, 1, 1, col_stats=stats[1])
        da = F.conv_igemm_dgrad(dy, w2, (128, 4, 4, 128), 3, 3, 1)
        return a, b, da

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


def test_flagship_step_launches_the_wide_halo_kernel_seven_times(monkeypatch):
    """ResNet-18, 32x32, batch 128: the four layer2 3x3 convolutions forward and the input gradients of the three
    stride-1 ones; the layer1 kernel still takes its eight GEMMs."""
    from baton_b200.models import resnet18
    from baton_b200.ops import load
    from baton_b200.ops import nn as bnn
    from baton_b200.parallel.arena import ParamArena

    calls = {"conv_halo": [], "conv_halo_wide": []}

    class Counting:
        def __init__(self, inner):
            self.inner = inner

        def __getattr__(self, name):
            fn = getattr(self.inner, name)
            if name not in calls:
                return fn

            def counted(*args):
                calls[name].append((args[3], args[4]) if name == "conv_halo_wide" else args[3])
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
    assert sorted(calls["conv_halo"]) == [False] * 4 + [True] * 4
    # (stride, dgrad): layer2.0.conv1 forward, three stride-1 forwards, three stride-1 input gradients
    assert sorted(calls["conv_halo_wide"]) == [(1, False)] * 3 + [(1, True)] * 3 + [(2, False)]
