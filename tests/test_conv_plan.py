"""The GEMM lowering of every convolution (``F.conv_plan``), pinned at the benchmark shapes (pure Python, no GPU):
training, its backward, the fused BatchNorm statistics and evaluation all take their lowering from this one plan,
so a change to it shows up here rather than as a silently different kernel."""
import pytest
import torch
from torch.nn import functional as TF

from baton_b200.models import resnet18, resnet50
from baton_b200.ops import functional as F
from baton_b200.ops import nn as bnn

BATCH = 128

# (conv, form, ho, wo, K, dgrad) of every convolution at batch 128 and 32x32 inputs
RESNET18 = [
    ("conv1", "im2col", 16, 16, 152, "col2im"),
    ("layer1.0.conv1", "implicit", 8, 8, 576, "implicit"),
    ("layer1.0.conv2", "implicit", 8, 8, 576, "implicit"),
    ("layer1.1.conv1", "implicit", 8, 8, 576, "implicit"),
    ("layer1.1.conv2", "implicit", 8, 8, 576, "implicit"),
    ("layer2.0.downsample.0", "implicit", 4, 4, 64, "implicit"),
    ("layer2.0.conv1", "implicit", 4, 4, 576, "implicit"),
    ("layer2.0.conv2", "implicit", 4, 4, 1152, "implicit"),
    ("layer2.1.conv1", "implicit", 4, 4, 1152, "implicit"),
    ("layer2.1.conv2", "implicit", 4, 4, 1152, "implicit"),
    ("layer3.0.downsample.0", "implicit", 2, 2, 128, "implicit"),
    ("layer3.0.conv1", "implicit", 2, 2, 1152, "implicit"),
    ("layer3.0.conv2", "implicit", 2, 2, 2304, "implicit"),
    ("layer3.1.conv1", "implicit", 2, 2, 2304, "implicit"),
    ("layer3.1.conv2", "implicit", 2, 2, 2304, "implicit"),
    ("layer4.0.downsample.0", "implicit", 1, 1, 256, "implicit"),
    ("layer4.0.conv1", "implicit", 1, 1, 2304, "implicit"),
    ("layer4.0.conv2", "centre", 1, 1, 512, "view"),
    ("layer4.1.conv1", "centre", 1, 1, 512, "view"),
    ("layer4.1.conv2", "centre", 1, 1, 512, "view"),
]

RESNET50 = [
    ("conv1", "im2col", 16, 16, 152, "col2im"),
    ("layer1.0.downsample.0", "pointwise", 8, 8, 64, "view"),
    ("layer1.0.conv1", "pointwise", 8, 8, 64, "view"),
    ("layer1.0.conv2", "implicit", 8, 8, 576, "implicit"),
    ("layer1.0.conv3", "pointwise", 8, 8, 64, "view"),
    ("layer1.1.conv1", "pointwise", 8, 8, 256, "view"),
    ("layer1.1.conv2", "implicit", 8, 8, 576, "implicit"),
    ("layer1.1.conv3", "pointwise", 8, 8, 64, "view"),
    ("layer1.2.conv1", "pointwise", 8, 8, 256, "view"),
    ("layer1.2.conv2", "implicit", 8, 8, 576, "implicit"),
    ("layer1.2.conv3", "pointwise", 8, 8, 64, "view"),
    ("layer2.0.downsample.0", "implicit", 4, 4, 256, "implicit"),
    ("layer2.0.conv1", "pointwise", 8, 8, 256, "view"),
    ("layer2.0.conv2", "implicit", 4, 4, 1152, "implicit"),
    ("layer2.0.conv3", "pointwise", 4, 4, 128, "view"),
    ("layer2.1.conv1", "pointwise", 4, 4, 512, "view"),
    ("layer2.1.conv2", "implicit", 4, 4, 1152, "implicit"),
    ("layer2.1.conv3", "pointwise", 4, 4, 128, "view"),
    ("layer2.2.conv1", "pointwise", 4, 4, 512, "view"),
    ("layer2.2.conv2", "implicit", 4, 4, 1152, "implicit"),
    ("layer2.2.conv3", "pointwise", 4, 4, 128, "view"),
    ("layer2.3.conv1", "pointwise", 4, 4, 512, "view"),
    ("layer2.3.conv2", "implicit", 4, 4, 1152, "implicit"),
    ("layer2.3.conv3", "pointwise", 4, 4, 128, "view"),
    ("layer3.0.downsample.0", "implicit", 2, 2, 512, "implicit"),
    ("layer3.0.conv1", "pointwise", 4, 4, 512, "view"),
    ("layer3.0.conv2", "implicit", 2, 2, 2304, "implicit"),
    ("layer3.0.conv3", "pointwise", 2, 2, 256, "view"),
    ("layer3.1.conv1", "pointwise", 2, 2, 1024, "view"),
    ("layer3.1.conv2", "implicit", 2, 2, 2304, "implicit"),
    ("layer3.1.conv3", "pointwise", 2, 2, 256, "view"),
    ("layer3.2.conv1", "pointwise", 2, 2, 1024, "view"),
    ("layer3.2.conv2", "implicit", 2, 2, 2304, "implicit"),
    ("layer3.2.conv3", "pointwise", 2, 2, 256, "view"),
    ("layer3.3.conv1", "pointwise", 2, 2, 1024, "view"),
    ("layer3.3.conv2", "implicit", 2, 2, 2304, "implicit"),
    ("layer3.3.conv3", "pointwise", 2, 2, 256, "view"),
    ("layer3.4.conv1", "pointwise", 2, 2, 1024, "view"),
    ("layer3.4.conv2", "implicit", 2, 2, 2304, "implicit"),
    ("layer3.4.conv3", "pointwise", 2, 2, 256, "view"),
    ("layer3.5.conv1", "pointwise", 2, 2, 1024, "view"),
    ("layer3.5.conv2", "implicit", 2, 2, 2304, "implicit"),
    ("layer3.5.conv3", "pointwise", 2, 2, 256, "view"),
    ("layer4.0.downsample.0", "implicit", 1, 1, 1024, "implicit"),
    ("layer4.0.conv1", "pointwise", 2, 2, 1024, "view"),
    ("layer4.0.conv2", "implicit", 1, 1, 4608, "implicit"),
    ("layer4.0.conv3", "pointwise", 1, 1, 512, "view"),
    ("layer4.1.conv1", "pointwise", 1, 1, 2048, "view"),
    ("layer4.1.conv2", "centre", 1, 1, 512, "view"),
    ("layer4.1.conv3", "pointwise", 1, 1, 512, "view"),
    ("layer4.2.conv1", "pointwise", 1, 1, 2048, "view"),
    ("layer4.2.conv2", "centre", 1, 1, 512, "view"),
    ("layer4.2.conv3", "pointwise", 1, 1, 512, "view"),
]

# (n, h, w, c, cout, kh, kw, stride, pad) -> (form, ho, wo, K, dgrad)
EDGES = [
    ((BATCH, 8, 8, 32, 64, 3, 3, 1, 1), ("im2col", 8, 8, 288, "col2im")),        # C % 64 != 0
    ((BATCH, 8, 8, 12, 64, 1, 1, 1, 0), ("im2col", 8, 8, 16, "col2im")),         # 1x1 with C % 8 != 0: K padded
    ((BATCH, 8, 8, 64, 128, 1, 1, 2, 0), ("implicit", 4, 4, 64, "implicit")),    # 1x1 stride 2
    ((BATCH, 8, 8, 24, 64, 1, 1, 2, 0), ("im2col", 4, 4, 24, "col2im")),         # 1x1 stride 2, C % 64 != 0
    ((BATCH, 8, 8, 64, 64, 1, 1, 1, 1), ("implicit", 10, 10, 64, "col2im")),     # 1x1 stride 1 with padding
    ((BATCH, 9, 9, 64, 64, 3, 3, 3, 1), ("implicit", 3, 3, 576, "col2im")),      # stride 3: no implicit dgrad
    ((BATCH, 1, 1, 4, 64, 3, 3, 1, 1), ("im2col", 1, 1, 40, "col2im")),          # 1x1 map, C % 8 != 0: no centre
    ((BATCH, 1, 1, 64, 64, 3, 3, 2, 1), ("centre", 1, 1, 64, "view")),           # centre tap at any stride
]


def _conv_inputs(model):
    """(name, conv, NHWC input shape at batch BATCH) of every convolution, in forward order."""
    seen = []
    hooks = [m.register_forward_pre_hook(lambda m, a, name=name: seen.append((name, m, a[0].shape[1:])))
             for name, m in model.named_modules() if isinstance(m, bnn.Conv2d)]
    with torch.no_grad():
        model.eval()(torch.zeros(2, 32, 32, 3))
    for h in hooks:
        h.remove()
    return [(name, m, (BATCH,) + tuple(shape)) for name, m, shape in seen]


@pytest.mark.parametrize("make, table", [(resnet18, RESNET18), (resnet50, RESNET50)], ids=["resnet18", "resnet50"])
def test_every_resnet_conv_keeps_its_lowering(make, table, monkeypatch):
    convs = _conv_inputs(make(10))
    assert [name for name, _, _ in convs] == [row[0] for row in table]
    stats_args = []
    monkeypatch.setattr(F, "gemm_stats_fusable", lambda M, N, K: stats_args.append((M, N, K)) or True)
    for (name, conv, shape), (_, form, ho, wo, K, dgrad) in zip(convs, table):
        x = torch.empty(shape, device="meta")
        plan = conv.plan(x)
        assert (plan.form, plan.ho, plan.wo, plan.K, plan.dgrad) == (form, ho, wo, K, dgrad), name
        assert plan.M == BATCH * ho * wo and plan.cout == conv.out_channels, name
        assert plan.tap == (4 if form == "centre" else None), name
        if form == "im2col":
            assert plan.K == conv.kp, name      # the zero-padded weights _w_bf16 hands the GEMM
        # the fused BatchNorm statistics are decided on the forward GEMM of the same plan
        conv.train()
        conv.bn_ws = torch.zeros(4 * conv.out_channels)
        stats_args.clear()
        ws = conv._fusable_stats(x)
        assert stats_args == [(plan.M, plan.cout, plan.K)], name
        assert ws.data_ptr() == conv.bn_ws.data_ptr() and ws.numel() == 2 * conv.out_channels, name


@pytest.mark.parametrize("geom, expect", EDGES)
def test_edge_shapes(geom, expect):
    plan = F.conv_plan(*geom)
    n, h, w, c, cout, kh, kw, stride, pad = geom
    assert (plan.form, plan.ho, plan.wo, plan.K, plan.dgrad) == expect
    assert plan.M == n * plan.ho * plan.wo
    assert (plan.n, plan.h, plan.w, plan.c, plan.cout, plan.kh, plan.kw, plan.stride, plan.pad) == geom


def test_im2col_k_is_the_one_padding_rule():
    assert F.im2col_k(7, 7, 3) == 152
    assert F.im2col_k(1, 1, 12) == 16
    assert F.im2col_k(3, 3, 64) == 576
    conv = bnn.Conv2d(3, 64, 7, 2, 3)
    assert (conv.k_true, conv.kp) == (147, F.im2col_k(7, 7, 3))


@pytest.mark.parametrize("geom", [g for g, _ in EDGES] + [(BATCH, 32, 32, 3, 64, 7, 7, 2, 3),
                                                          (BATCH, 4, 4, 16, 32, 3, 3, 2, 1)])
def test_plan_gemm_computes_the_convolution(geom):
    """The plan's forward GEMM ``A [M, K] x B [Cout, K]^T``, built on the CPU in float64 -- ``x.view(M, C)`` for the
    centre and pointwise forms, im2col zero-padded to ``K`` otherwise, ``plan.weight`` as B -- is the convolution."""
    _, h, w, c, cout, kh, kw, stride, pad = geom
    n = 2
    plan = F.conv_plan(n, h, w, c, cout, kh, kw, stride, pad)
    g = torch.Generator().manual_seed(0)
    x = torch.randn(n, h, w, c, generator=g, dtype=torch.float64)
    wt = torch.randn(cout, c, kh, kw, generator=g, dtype=torch.float64)
    w2d = wt.permute(0, 2, 3, 1).reshape(cout, kh * kw * c)          # channels_last [Cout, kh*kw*C]
    if plan.form in ("centre", "pointwise"):
        a = x.reshape(plan.M, c)
    else:
        cols = TF.unfold(x.permute(0, 3, 1, 2), (kh, kw), padding=pad, stride=stride)    # [n, C*kh*kw, L]
        a = cols.view(n, c, kh * kw, -1).permute(0, 3, 2, 1).reshape(-1, kh * kw * c)
        a, w2d = TF.pad(a, (0, plan.K - kh * kw * c)), TF.pad(w2d, (0, plan.K - kh * kw * c))
    b = plan.weight(w2d)
    assert a.shape == (plan.M, plan.K) and b.shape == (cout, plan.K)
    ref = TF.conv2d(x.permute(0, 3, 1, 2), wt, stride=stride, padding=pad).permute(0, 2, 3, 1)
    assert ref.shape == (n, plan.ho, plan.wo, cout)
    torch.testing.assert_close(a @ b.T, ref.reshape(plan.M, cout))
