"""Vision Transformers on the CPU: torchvision's state_dict and function, construction errors, configuration, FedPer
keys and a few local-SGD steps with the DeiT augmentation."""
import pytest
import torch
from torchvision.models.vision_transformer import VisionTransformer as TV

from baton_b200.models import VisionTransformer, vit_small, vit_tiny


def _pair(image=16, patch=4, layers=2, heads=2, dim=128, mlp=256, classes=5):
    return VisionTransformer(image, patch, layers, heads, dim, mlp, classes), TV(image, patch, layers, heads, dim, mlp,
                                                                                num_classes=classes)


@pytest.mark.parametrize("ctor,tv_args,n_floats", [(vit_tiny, (32, 4, 12, 3, 192, 768), 5362762),
                                                   (vit_small, (32, 4, 12, 6, 384, 1536), 21342346), (None, None, None)])
def test_state_dict_is_torchvisions(ctor, tv_args, n_floats):
    if ctor is None:
        m, tv = _pair()
    else:
        m, tv = ctor(10), TV(*tv_args, num_classes=10)
    a, b = m.state_dict(), tv.state_dict()
    assert list(a) == list(b)
    assert all(a[k].shape == b[k].shape for k in a)
    if n_floats is not None:
        assert sum(v.numel() for v in a.values()) == n_floats
    if ctor is vit_tiny:
        assert len(a) == 152
    m.load_state_dict(b, strict=True)
    tv.load_state_dict(a, strict=True)
    assert not list(m.buffers()) and all(p.requires_grad for p in m.parameters())


def test_initialisation_follows_torchvision():
    m = vit_tiny(10)
    assert not m.class_token.any() and not m.heads.head.weight.any() and not m.heads.head.bias.any()
    assert abs(float(m.encoder.pos_embedding.detach().std()) - 0.02) < 2e-3
    blk = m.encoder.layers.encoder_layer_0
    assert not blk.self_attention.in_proj_bias.any() and not blk.self_attention.out_proj.bias.any()
    assert float(blk.mlp[0].bias.abs().max()) < 1e-4
    assert m.conv_proj.weight.is_contiguous(memory_format=torch.channels_last)
    assert abs(float(m.conv_proj.weight.detach().std()) / (1 / 48) ** 0.5 - 1) < 0.05


def test_cpu_forward_and_gradients_match_torchvision():
    torch.manual_seed(0)
    m, tv = _pair()
    for p in tv.parameters():
        torch.nn.init.normal_(p, std=0.1)
    m.load_state_dict(tv.state_dict())
    x = torch.randn(3, 3, 16, 16, requires_grad=True)
    xn = x.detach().permute(0, 2, 3, 1).contiguous().requires_grad_()
    ref, out = tv(x), m(xn)
    assert float((out - ref).abs().max()) <= 1e-5 * float(ref.abs().max())
    ref.square().sum().backward()
    out.square().sum().backward()
    assert float((xn.grad - x.grad.permute(0, 2, 3, 1)).abs().max()) <= 1e-5 * float(x.grad.abs().max())
    theirs = dict(tv.named_parameters())
    for k, p in m.named_parameters():
        g = theirs[k].grad
        assert float((p.grad - g).abs().max()) <= 1e-5 * float(g.abs().max()), k


@pytest.mark.parametrize("kw,msg", [(dict(image_size=30, patch_size=4), "divisible"),
                                    (dict(image_size=64, patch_size=4), "tokens"),
                                    (dict(image_size=224, patch_size=16), "tokens"),
                                    (dict(num_heads=4), "must be 64"),
                                    (dict(num_layers=0), "positive")])
def test_construction_errors(kw, msg):
    args = dict(image_size=32, patch_size=4, num_layers=1, num_heads=3, hidden_dim=192, mlp_dim=384, num_classes=10)
    args.update(kw)
    with pytest.raises(ValueError, match=msg):
        VisionTransformer(**args)


def test_build_model_and_config():
    from baton_b200.config import FederationConfig
    from baton_b200.demo import build_model
    assert build_model("vit_tiny").name == "vit_tiny" and build_model("vit_small").name == "vit_small"
    for backend in ("http", "fused", "nccl"):
        FederationConfig(model="vit_tiny", backend=backend)
        FederationConfig(model="vit_small", backend=backend)
    with pytest.raises(ValueError, match="dropout"):
        FederationConfig(model="vit_tiny", dropout=0.1)
    with pytest.raises(ValueError, match="LoRA"):
        FederationConfig(model="vit_tiny", lora_r=8)
    with pytest.raises(ValueError, match="dropout"):
        build_model("vit_tiny", dropout=0.1)


def test_local_keys_and_tile_flags():
    from baton_b200.parallel.features import check_features
    from baton_b200.parallel.personal import resolve_local_keys
    m, _ = _pair()
    assert resolve_local_keys(m, "head") == ["heads.head.weight", "heads.head.bias"]
    with pytest.raises(ValueError):
        resolve_local_keys(m, "bn")
    with pytest.raises(ValueError, match="Vision Transformer with tile_flags"):
        check_features(tile_flags=True, vit=True)
    check_features(tile_flags=True)
    check_features(vit=True)


def test_payload_is_a_plain_state_dict():
    m, tv = _pair()
    sd = m.state_dict()
    assert all(v.dtype == torch.float32 for v in sd.values())
    tv.load_state_dict(sd, strict=True)


def test_local_sgd_with_crop_flip_and_mixup_cutmix_lowers_the_loss():
    from baton_b200.data import dirichlet_label_shards, image_shard
    torch.manual_seed(0)
    spec = dirichlet_label_shards(1, 10, 64, 0.5, 0)[0]
    X, y = image_shard(spec, seed=0, size=16)
    m = VisionTransformer(16, 4, 1, 1, 64, 128, 10)
    hist = m.train(X, y, n_epoch=6, lr=3e-3, batch_size=32, optimizer="adamw", augment="crop_flip",
                   mix="mixup_cutmix", label_smoothing=0.1)
    assert all(h == h for h in hist) and hist[-1] < hist[0], hist
