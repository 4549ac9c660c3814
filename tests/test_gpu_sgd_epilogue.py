"""Optimizer epilogue of the weight-gradient GEMMs: SGD applied in the GEMM epilogue plus the leftover segment pass must
give the same bits as "accumulate the gradient into a zeroed buffer, then one fused_sgd pass over the arena"."""
import pytest
import torch

pytestmark = pytest.mark.gpu

BF16 = torch.bfloat16

# ResNet-18 on 32x32 inputs, batch 128: (input NHWC, kernel, stride, pad, Cout)
SHAPES = {
    "igemm_layer3": ((128, 4, 4, 128), 3, 2, 1, 256),     # layer3.0.conv1
    "shortcut_layer4": ((128, 2, 2, 256), 1, 2, 0, 512),  # layer4.0.downsample: 1x1 stride 2
    "centre_layer4": ((128, 1, 1, 512), 3, 1, 1, 512),    # layer4.0.conv2: 3x3 on a 1x1 map, centre tap only
}
HYPER = [(0.0, False, 0.0), (0.0, False, 5e-4), (0.9, False, 0.0), (0.9, False, 5e-4), (0.9, True, 0.0),
         (0.9, True, 5e-4)]


@pytest.fixture(scope="module")
def F():
    from baton_b200.ops import functional
    return functional


def _bits(t):
    return t.view(torch.int16) if t.dtype == BF16 else t.view(torch.int32)


@pytest.mark.parametrize("mu,nesterov,wd", HYPER)
@pytest.mark.parametrize("shape", sorted(SHAPES))
def test_epilogue_sgd_matches_accumulate_then_fused_sgd(F, shape, mu, nesterov, wd):
    torch.manual_seed(0)
    dev = torch.device("cuda:0")
    xs, k, stride, pad, cout = SHAPES[shape]
    n_img, h, _, c = xs
    ho = F.conv_out_size(h, k, stride, pad)
    x = torch.randn(xs, device=dev).to(BF16)
    dy = torch.randn(n_img * ho * ho, cout, device=dev).to(BF16)
    centre = shape.startswith("centre")
    numel = cout * k * k * c
    off = 1024                                              # parameters with a gradient before and after the conv weight
    n = off + numel + 1032
    theta0 = torch.randn(n, device=dev) * 0.05
    mom0 = torch.randn(n, device=dev) * 0.01 if mu else None
    hyper = torch.tensor([0.05, mu, wd, 0.0], device=dev)

    def state():
        grad = torch.zeros(n, device=dev)
        grad[:off] = torch.linspace(-1.0, 1.0, off, device=dev)            # gradients of the other parameters
        grad[off + numel:] = torch.linspace(-0.5, 0.5, n - off - numel, device=dev)
        theta = theta0.clone()
        return theta, grad, theta.to(BF16), mom0.clone() if mom0 is not None else None

    def out_view(grad):
        w2d = grad[off: off + numel].view(cout, k * k * c)
        return w2d.view(cout, k * k, c)[:, (k * k) // 2, :] if centre else w2d

    def wgrad(out2d, sgd=None):
        if centre:
            return F.gemm(dy, x.view(n_img, c), a_mn=True, b_mn=True, out=out2d, accumulate=True, sgd=sgd) is not None
        return F.conv_igemm_wgrad_(dy, x, out2d, k, k, stride, pad, sgd=sgd)

    theta_r, grad_r, wb_r, mom_r = state()
    assert wgrad(out_view(grad_r))
    assert grad_r[off: off + numel].abs().max() > 0
    F.fused_sgd(theta_r, grad_r, hyper, mom_r, wb_r, zero_grad=True, nesterov=nesterov)

    theta, grad, wb, mom = state()
    out2d = out_view(grad)
    assert wgrad(out2d, F.sgd_epilogue_args(theta, grad, out2d, hyper, mom, wb, nesterov)), "epilogue declined"
    assert (grad[off: off + numel] == 0).all(), "the optimizer epilogue must not write the gradient"
    fused = [(off + (4 * c if centre else 0), out2d.shape[0], out2d.shape[1], out2d.stride(0))]
    segs = F.sgd_segments(n, fused, [(off, numel)] if centre else [])
    F.fused_sgd_segments(theta, grad, hyper, torch.tensor(segs, dtype=torch.int64, device=dev), mom, wb,
                         nesterov=nesterov)
    torch.cuda.synchronize()

    assert not torch.equal(theta_r, theta0)
    assert torch.equal(_bits(theta), _bits(theta_r))
    assert torch.equal(_bits(wb), _bits(wb_r))
    if mom is not None:
        assert torch.equal(_bits(mom), _bits(mom_r))
    assert (grad == 0).all() and (grad_r == 0).all()


def test_nograd_segment_applies_weight_decay(F):
    """Parameters whose gradient is identically zero: updated with g = 0 when weight decay is on, skipped (left exactly
    as they are) when the update is the identity; decided from the device hyper-parameters."""
    dev = torch.device("cuda:0")
    n = 3 * 8192 + 40
    theta0 = torch.randn(n, device=dev)
    segs = torch.tensor([[0, 8192, 1], [8192, 8192, 0], [16384, 8232, 1]], dtype=torch.int64, device=dev)
    for wd in (0.0, 5e-4):
        hyper = torch.tensor([0.1, 0.0, wd, 0.0], device=dev)
        theta, grad, wb = theta0.clone(), torch.full((n,), float("nan"), device=dev), theta0.to(BF16)
        grad[8192:16384] = 1.0
        F.fused_sgd_segments(theta, grad, hyper, segs, None, wb)
        ng = torch.cat([torch.arange(0, 8192), torch.arange(16384, n)]).to(dev)
        want = theta0[ng] - 0.1 * (wd * theta0[ng])
        assert torch.equal(theta[ng], theta0[ng]) if wd == 0 else torch.allclose(theta[ng], want, rtol=0, atol=1e-6)
        assert torch.isnan(grad[ng]).all(), "a no-grad segment must not read or write the gradient"
        assert (grad[8192:16384] == 0).all()
        assert torch.allclose(theta[8192:16384], theta0[8192:16384] - 0.1 * (1.0 + wd * theta0[8192:16384]))
        assert torch.equal(wb, theta.to(BF16))
