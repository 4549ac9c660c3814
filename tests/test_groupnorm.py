"""GroupNorm ResNets on the host: the CPU layer against float64 ``group_norm``, the torchvision correspondence of the
``state_dict``, construction errors, the model registry and one portable engine round."""
import math

import pytest
import torch
from torch import nn
from torch.nn import functional as TF

from baton_b200.config import FederationConfig
from baton_b200.demo import build_model
from baton_b200.models import resnet18, resnet50
from baton_b200.ops import nn as bnn
from baton_b200.parallel.engine import FederatedEngine

tv = pytest.importorskip("torchvision.models")


def _reference(x, residual, gn, relu):
    """float64 ``relu(group_norm(x) + residual)`` on the NCHW permute of an NHWC tensor."""
    y = TF.group_norm(x.double().permute(0, 3, 1, 2), gn.num_groups, gn.weight.double(), gn.bias.double(),
                      gn.eps).permute(0, 2, 3, 1)
    if residual is not None:
        y = y + residual.double()
    return TF.relu(y) if relu else y


@pytest.mark.parametrize("groups,c,hw", [(1, 8, 5), (2, 64, 4), (32, 64, 3), (4, 12, 7)])
@pytest.mark.parametrize("residual", [False, True])
@pytest.mark.parametrize("relu", [False, True])
def test_cpu_layer_matches_float64_group_norm(groups, c, hw, residual, relu):
    g = torch.Generator().manual_seed(groups * 1000 + c + hw)
    gn = bnn.GroupNorm(groups, c, relu=relu)
    with torch.no_grad():
        gn.weight.copy_(torch.randn(c, generator=g))
        gn.bias.copy_(torch.randn(c, generator=g))
    x = torch.randn(3, hw, hw, c, generator=g) * 4 + 2
    r = torch.randn(3, hw, hw, c, generator=g) if residual else None
    y = gn(x, r)
    assert y.shape == x.shape
    torch.testing.assert_close(y.double(), _reference(x, r, gn, relu), rtol=1e-5, atol=1e-5)


@pytest.mark.parametrize("bad", [0, -2, 3, 2.0, True, None])
def test_groups_must_be_a_positive_int_dividing_the_channels(bad):
    with pytest.raises(ValueError):
        bnn.GroupNorm(bad, 64)


def test_resnet_rejects_bad_groups_and_norm():
    with pytest.raises(ValueError):
        resnet18(10, norm="group", groups=3)        # 3 does not divide 64
    with pytest.raises(ValueError):
        resnet18(10, norm="layer")


def _floats(sd):
    return sum(v.numel() for v in sd.values() if v.is_floating_point())


@pytest.mark.parametrize("depth", [18, 50])
@pytest.mark.parametrize("groups", [2, 32])
def test_state_dict_round_trips_with_torchvision(depth, groups):
    ours = (resnet18 if depth == 18 else resnet50)(10, norm="group", groups=groups)
    ref = getattr(tv, "resnet{}".format(depth))(num_classes=10, norm_layer=lambda c: nn.GroupNorm(groups, c))
    assert not list(ours.buffers())
    torch.manual_seed(0)
    with torch.no_grad():
        for p in ref.parameters():
            p.copy_(torch.randn_like(p))
    ours.load_state_dict(ref.state_dict(), strict=True)
    back = getattr(tv, "resnet{}".format(depth))(num_classes=10, norm_layer=lambda c: nn.GroupNorm(groups, c))
    back.load_state_dict(ours.state_dict(), strict=True)
    for k, v in ref.state_dict().items():
        assert torch.equal(back.state_dict()[k], v), k
    if depth == 18:
        sd = ours.state_dict()
        assert len(sd) == 62 and _floats(sd) == 11_181_642
        bn = resnet18(10).state_dict()
        assert len(bn) == 122 and _floats(bn) == 11_191_242


def test_group_forward_matches_torchvision_on_cpu():
    torch.manual_seed(0)
    ours = resnet18(10, norm="group", groups=2)
    ref = tv.resnet18(num_classes=10, norm_layer=lambda c: nn.GroupNorm(2, c))
    with torch.no_grad():
        for p in ref.parameters():
            p.copy_(torch.randn_like(p) * 0.1)
    ours.load_state_dict(ref.state_dict())
    x = torch.randn(4, 32, 32, 3)
    torch.testing.assert_close(ours(x), ref(x.permute(0, 3, 1, 2)), rtol=1e-4, atol=1e-4)


def test_zero_init_of_each_blocks_last_norm_weight():
    m = resnet18(10, norm="group")
    for blk in (b for layer in (m.layer1, m.layer2, m.layer3, m.layer4) for b in layer):
        assert isinstance(blk.bn2, bnn.GroupNorm) and not blk.bn2.weight.any()
        assert blk.bn1.weight.eq(1).all()
    m50 = resnet50(10, norm="group")
    assert not m50.layer1[0].bn3.weight.any()
    assert isinstance(m50.layer1[0].downsample[1], bnn.GroupNorm)


def test_batch_norm_model_is_unchanged():
    torch.manual_seed(0)
    a = resnet18(10)
    torch.manual_seed(0)
    b = resnet18(10, norm="batch")
    assert a.name == "resnet18" and b.norm == "batch"
    for (ka, va), (kb, vb) in zip(a.state_dict().items(), b.state_dict().items()):
        assert ka == kb and torch.equal(va, vb)
    assert all(isinstance(m, bnn.BatchNorm2d) for n, m in a.named_modules() if n.endswith("bn1"))


def test_registry_builds_group_norm_resnets():
    m = build_model("resnet18_gn")
    assert m.name == "resnet18_gn" and m.norm == "group"
    assert all(g.num_groups == 2 for g in m.modules() if isinstance(g, bnn.GroupNorm))
    assert not any(isinstance(g, bnn.BatchNorm2d) for g in m.modules())
    assert build_model("resnet50_gn").fc.out_features == 1000
    cfg = FederationConfig.from_json(FederationConfig(model="resnet18_gn").to_json())
    assert build_model(cfg.model).name == "resnet18_gn"


def _shard(cid, n=16, classes=10):
    g = torch.Generator().manual_seed(100 + cid)
    return torch.randn(n, 32, 32, 3, generator=g), torch.randint(0, classes, (n,), generator=g)


def test_portable_engine_round_on_a_group_norm_resnet():
    torch.manual_seed(0)
    model = resnet18(10, norm="group")
    before = {k: v.clone() for k, v in model.state_dict().items()}
    eng = FederatedEngine(model, "cpu", backend="nccl", lr=0.05, batch_size=8, logical_clients=2, seed=1)
    res = eng.run_round(lambda cid: _shard(cid), n_epoch=1)
    assert all(math.isfinite(v) for v in eng.global_loss(1))
    after = eng.state_dict()
    assert set(after) == set(before)
    assert any(not torch.equal(after[k].cpu(), before[k]) for k in before if k.endswith("bn1.bias"))
    assert res is not None


def test_fedbn_local_keys_match_no_group_norm_entry():
    with pytest.raises(ValueError, match="matches no float state_dict entry"):
        FederatedEngine(resnet18(10, norm="group"), "cpu", backend="nccl", local_keys="bn")
