"""Image-tile 3x3 convolution (`conv_smallmap`, csrc/conv_halo.cu in image mode; ResNet-18 layer3 shapes) against
the im2col-mode implicit GEMM with cluster split-K 1 and against fp32 torch."""
import pytest
import torch

from baton_b200.ops import functional as F

pytestmark = pytest.mark.gpu
BF16 = torch.bfloat16
COUT = 256

# (gathered channels, input size, stride): layer3.0.conv1 (stride 2, 128 -> 256, 4x4 -> 2x2) and the stride-1 layer3
# convolutions (256 -> 256, 2x2)
LAYER3_S2, LAYER3 = (128, 4, 2), (256, 2, 1)
# (batch, cluster size): 2x2 output maps, 16 images per 64-row tile.  128 and 126 (a partial last tile: 14 images)
# give 8 tiles, which every cluster size divides; 3 and 1 give one tile.
CASES = [(n, mc) for n in (128, 126) for mc in (1, 2, 4, 8)] + [(3, 1), (1, 1)]


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


@pytest.mark.parametrize("cin,h,stride,n,mc,bn", [f + c + (32,) for f in (LAYER3_S2, LAYER3) for c in CASES] +
                         [LAYER3_S2 + c + (64,) for c in ((128, 4), (126, 8), (3, 1))])
def test_forward_matches_im2col_path_and_torch(cin, h, stride, n, mc, bn):
    x, w2d = _data(n, h, cin, COUT)
    assert F.smallmap_eligible(3, 3, stride, 1, cin, h, h)
    y_old = F.conv_igemm_fwd(x, w2d, 3, 3, stride, 1, path="im2col", cluster_k=1)
    y = F.conv_igemm_fwd(x, w2d, 3, 3, stride, 1, path="smallmap", mc=mc, bn=bn)
    torch.cuda.synchronize()
    # all nine taps in the im2col k order (tap-major, then channel block, then 4 x k16), one pass over K: the same bits
    assert torch.equal(y, y_old)
    ref = torch.nn.functional.conv2d(x.float().permute(0, 3, 1, 2), _w4(w2d, cin), stride=stride, padding=1)
    _close(y, ref.permute(0, 2, 3, 1).reshape(-1, COUT))


@pytest.mark.parametrize("n,mc", CASES)
def test_dgrad_matches_im2col_path_and_torch(n, mc):
    dy, _ = _data(n, 2, COUT, COUT, seed=1)
    _, w2d = _data(1, 2, COUT, COUT, seed=2)
    dx_old = F.conv_igemm_dgrad(dy, w2d, (n, 2, 2, COUT), 3, 3, 1, path="im2col", cluster_k=1)
    dx = F.conv_igemm_dgrad(dy, w2d, (n, 2, 2, COUT), 3, 3, 1, path="smallmap", mc=mc)
    torch.cuda.synchronize()
    assert torch.equal(dx, dx_old)
    ref = torch.nn.grad.conv2d_input((n, COUT, 2, 2), _w4(w2d, COUT), dy.float().permute(0, 3, 1, 2), padding=1)
    _close(dx, ref.permute(0, 2, 3, 1))


@pytest.mark.parametrize("cin,h,stride,n,mc,bn", [f + c + (32,) for f in (LAYER3_S2, LAYER3)
                                                  for c in ((128, 4), (126, 8), (3, 1))] +
                         [LAYER3_S2 + (126, 2, 64)])
def test_fused_column_statistics(cin, h, stride, n, mc, bn):
    x, w2d = _data(n, h, cin, COUT, seed=3)
    stats = torch.zeros(2 * COUT, device="cuda")
    y = F.conv_igemm_fwd(x, w2d, 3, 3, stride, 1, col_stats=stats, path="smallmap", mc=mc, bn=bn)
    torch.cuda.synchronize()
    yf = y.float()
    torch.testing.assert_close(stats[:COUT], yf.sum(0), rtol=1e-4, atol=1e-2)
    torch.testing.assert_close(stats[COUT:], (yf * yf).sum(0), rtol=1e-4, atol=1e-2)


def test_default_dispatch_takes_the_image_tile_kernel():
    x, w2d = _data(128, 2, COUT, COUT, seed=8)
    y = F.conv_igemm_fwd(x, w2d, 3, 3, 1, 1)
    y_small = F.conv_igemm_fwd(x, w2d, 3, 3, 1, 1, path="smallmap")
    torch.cuda.synchronize()
    assert torch.equal(y, y_small)


def test_graph_captured_layer3_chain_matches_eager():
    """layer3.0.conv1 and conv2 forward and conv2's input gradient, captured into one graph (PDL edges, clusters)."""
    x, w1 = _data(128, 4, 128, COUT, seed=5)
    _, w2 = _data(1, 2, COUT, COUT, seed=6)
    dy, _ = _data(128, 2, COUT, COUT, seed=7)
    stats = torch.zeros(2, 2 * COUT, device="cuda")

    def chain():
        stats.zero_()
        a = F.conv_igemm_fwd(x, w1, 3, 3, 2, 1, col_stats=stats[0])
        b = F.conv_igemm_fwd(a.view(128, 2, 2, COUT), w2, 3, 3, 1, 1, col_stats=stats[1])
        da = F.conv_igemm_dgrad(dy, w2, (128, 2, 2, COUT), 3, 3, 1)
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


def test_flagship_step_launches_the_image_tile_kernel_seven_times(monkeypatch):
    """ResNet-18, 32x32, batch 128: the four layer3 3x3 convolutions forward and the input gradients of the three
    stride-1 ones."""
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
            if name != "conv_smallmap":
                return fn

            def counted(src, w, out, stride, dgrad, mc, bn, col_stats):
                calls.append((src.shape[3], stride, dgrad))
                return fn(src, w, out, stride, dgrad, mc, bn, col_stats)
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
    assert sorted(calls) == sorted([(128, 2, False)] + [(256, 1, False)] * 3 + [(256, 1, True)] * 3)
