"""CPU checks of the image-tile kernel's dispatch rule (layer3 of ResNet-18 on 32x32 inputs) beside the halo rule."""
import pytest

from baton_b200.ops import functional as F

# ResNet-18 on 32x32 inputs: (name, Cin, Cout, k, stride, pad, input size); stem 7x7/2 -> 16x16, max-pool -> 8x8
RESNET18_32 = (
    [("conv1", 3, 64, 7, 2, 3, 32)]
    + [("layer1.{}.conv{}".format(b, c), 64, 64, 3, 1, 1, 8) for b in range(2) for c in (1, 2)]
    + [("layer2.0.conv1", 64, 128, 3, 2, 1, 8), ("layer2.0.conv2", 128, 128, 3, 1, 1, 4),
       ("layer2.0.downsample", 64, 128, 1, 2, 0, 8), ("layer2.1.conv1", 128, 128, 3, 1, 1, 4),
       ("layer2.1.conv2", 128, 128, 3, 1, 1, 4)]
    + [("layer3.0.conv1", 128, 256, 3, 2, 1, 4), ("layer3.0.conv2", 256, 256, 3, 1, 1, 2),
       ("layer3.0.downsample", 128, 256, 1, 2, 0, 4), ("layer3.1.conv1", 256, 256, 3, 1, 1, 2),
       ("layer3.1.conv2", 256, 256, 3, 1, 1, 2)]
    + [("layer4.0.conv1", 256, 512, 3, 2, 1, 2), ("layer4.0.conv2", 512, 512, 3, 1, 1, 1),
       ("layer4.0.downsample", 256, 512, 1, 2, 0, 2), ("layer4.1.conv1", 512, 512, 3, 1, 1, 1),
       ("layer4.1.conv2", 512, 512, 3, 1, 1, 1)]
)


def _picked(path_args, halo_args):
    return F._conv_path(None, F.halo_eligible(*halo_args), F.smallmap_eligible(*path_args))


def test_flagship_shapes_select_exactly_the_layer3_gemms():
    fwd = [name for name, cin, cout, k, s, p, h in RESNET18_32
           if _picked((k, k, s, p, cin, h, h), (k, k, s, p, cin, h, h)) == "smallmap" and cout % F.SMALLMAP_BN == 0]
    # the input gradient gathers dy (Cout channels) over the input image; the stem's is never computed
    dgrad = [name for name, _, cout, k, s, p, h in RESNET18_32[1:]
             if _picked((k, k, s, p, cout, h, h, None, True), (k, k, s, p, cout, h, h, None, True)) == "smallmap"]
    assert fwd == ["layer3.0.conv1", "layer3.0.conv2", "layer3.1.conv1", "layer3.1.conv2"]
    assert dgrad == ["layer3.0.conv2", "layer3.1.conv1", "layer3.1.conv2"]


def test_no_shape_is_admitted_by_both_rules():
    for _, cin, cout, k, s, p, h in RESNET18_32:
        for c, dgrad in ((cin, False), (cout, True)):
            assert not (F.halo_eligible(k, k, s, p, c, h, h, dgrad=dgrad) and
                        F.smallmap_eligible(k, k, s, p, c, h, h, dgrad=dgrad))


# args: (kh, kw, stride, pad, gathered channels, h, w[, affine, dgrad])
@pytest.mark.parametrize("args,ok", [
    ((3, 3, 1, 1, 256, 2, 2), True),                 # layer3 stride 1, forward
    ((3, 3, 1, 1, 256, 2, 2, None, True), True),     # and input gradient
    ((3, 3, 2, 1, 128, 4, 4), True),                 # layer3.0.conv1
    ((3, 3, 2, 1, 128, 4, 4, None, True), False),    # stride-2 input gradients have their own kernel
    ((3, 3, 1, 1, 256, 4, 4), True),                 # four 4x4 images per tile
    ((3, 3, 1, 1, 256, 1, 1), True),                 # 64 1x1 images (the "centre" plan never calls it)
    ((3, 3, 2, 1, 128, 3, 3), True),                 # odd input: row / column 3 of the taps is outside
    ((3, 3, 2, 1, 256, 2, 2), False),                # layer4.0.conv1: out of scope
    ((3, 3, 1, 1, 128, 2, 2), False),                # the halo kernel's form
    ((3, 3, 2, 1, 64, 4, 4), False),                 # the halo kernel's form
    ((3, 3, 1, 1, 512, 1, 1), False),
    ((3, 3, 1, 0, 256, 2, 2), False),                # not "same"
    ((1, 1, 1, 0, 256, 2, 2), False),
    ((1, 1, 2, 0, 128, 4, 4), False),
    ((3, 3, 1, 1, 256, 6, 6), False),                # 64 % 36 != 0
    ((3, 3, 1, 1, 256, 8, 16), False),               # 128 pixels: a 64-row tile holds no whole image
])
def test_smallmap_rule(args, ok):
    assert F.smallmap_eligible(*args) is ok


def test_smallmap_rule_declines_the_affine_epilogue():
    for args in ((3, 3, 1, 1, 256, 2, 2), (3, 3, 2, 1, 128, 4, 4)):
        assert not F.smallmap_eligible(*args, affine={"scale": None}), args


def test_smallmap_smem_bytes():
    # layer3 stride 1: four 16 x 2x2 x 128 B image boxes (8 KB each), 36 slots of 32 x 64 bf16 (4 KB), 37 mbarriers
    # padded to 48, statistics of 32 columns, the zero line and the realignment
    assert F.smallmap_smem_bytes(2, 2) == 4 * 8192 + 36 * 4096 + 48 * 8 + 512 + 128 + 1024
    # layer3.0.conv1: two 16 x 4x4 x 128 B boxes (32 KB each), 18 slots
    assert F.smallmap_smem_bytes(4, 4, c=128, stride=2) == 2 * 32768 + 18 * 4096 + 32 * 8 + 512 + 128 + 1024
    # 64 columns fit at the stride-2 form only: 36 slots of 8 KB alone are 288 KB
    assert F.smallmap_smem_bytes(4, 4, c=128, stride=2, bn=64) <= 227 * 1024
    assert F.smallmap_smem_bytes(2, 2, bn=64) > 227 * 1024
    for name, cin, cout, k, s, p, h in RESNET18_32:
        for c, dgrad in ((cin, False), (cout, True)):
            if F.smallmap_eligible(k, k, s, p, c, h, h, dgrad=dgrad):
                assert F.smallmap_smem_bytes(h, h, c, s) <= 227 * 1024, name
    for h in (1, 2, 4, 8):
        assert F.smallmap_smem_bytes(h, h) <= 227 * 1024
        assert F.smallmap_smem_bytes(2 * h, 2 * h, c=128, stride=2) <= 227 * 1024


def test_forced_smallmap_path_is_checked():
    with pytest.raises(ValueError):
        F._conv_path("smallmap", True, False)
    with pytest.raises(ValueError):
        F._conv_path("smallmap", False, F.smallmap_eligible(3, 3, 2, 1, 256, 2, 2))
    assert F._conv_path(None, False, True) == "smallmap"
    assert F._conv_path(None, True, True) == "halo"
    assert F._conv_path("im2col", False, True) == "im2col"
    assert F._conv_path("smallmap", False, True) == "smallmap"
