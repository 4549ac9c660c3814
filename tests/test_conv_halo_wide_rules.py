"""CPU checks of the wide-channel halo-kernel dispatch rule (layer2 of ResNet-18 on 32x32 inputs)."""
import pytest

from baton_b200.ops import functional as F
from test_conv_halo_rules import RESNET18_32


def test_flagship_shapes_select_exactly_the_layer2_gemms():
    fwd = [name for name, cin, _, k, s, p, h in RESNET18_32 if F.halo_wide_eligible(k, k, s, p, cin, h, h)]
    # the input gradient gathers dy (Cout channels) over the input image; the stem's is never computed
    dgrad = [name for name, _, cout, k, s, p, h in RESNET18_32[1:]
             if F.halo_wide_eligible(k, k, s, p, cout, h, h, dgrad=True)]
    assert fwd == ["layer2.0.conv1", "layer2.0.conv2", "layer2.1.conv1", "layer2.1.conv2"]
    assert dgrad == ["layer2.0.conv2", "layer2.1.conv1", "layer2.1.conv2"]


def test_the_two_halo_rules_never_overlap():
    for name, cin, cout, k, s, p, h in RESNET18_32:
        for c in (cin, cout):
            assert not (F.halo_eligible(k, k, s, p, c, h, h) and F.halo_wide_eligible(k, k, s, p, c, h, h)), name


@pytest.mark.parametrize("args,kw,ok", [
    ((3, 3, 1, 1, 128, 4, 4), {}, True),
    ((3, 3, 1, 1, 128, 4, 4), {"dgrad": True}, True),
    ((3, 3, 2, 1, 64, 8, 8), {}, True),
    ((3, 3, 2, 1, 64, 8, 8), {"dgrad": True}, False),     # stride-2 input gradients have their own kernel
    ((3, 3, 1, 1, 128, 2, 2), {}, True),
    ((3, 3, 1, 1, 128, 8, 8), {}, True),
    ((3, 3, 2, 1, 64, 4, 4), {}, True),                   # 2x2 outputs, 16 images per tile
    ((3, 3, 2, 1, 64, 16, 16), {}, True),                 # one 8x8 output image per tile
    ((3, 3, 1, 1, 64, 8, 8), {}, False),                  # one channel block: halo_eligible's
    ((3, 3, 1, 1, 256, 2, 2), {}, False),                 # four channel blocks: 36 k-tiles do not fit
    ((3, 3, 2, 1, 128, 4, 4), {}, False),
    ((3, 3, 1, 0, 128, 4, 4), {}, False),
    ((1, 1, 1, 0, 128, 4, 4), {}, False),
    ((3, 3, 1, 1, 128, 6, 6), {}, False),                 # 64 % 36 != 0
    ((3, 3, 2, 1, 64, 32, 32), {}, False),                # 256 output pixels: a 64-row tile holds no whole image
])
def test_halo_wide_rule(args, kw, ok):
    assert F.halo_wide_eligible(*args, **kw) is ok


def test_halo_wide_rule_declines_the_affine_epilogue():
    assert not F.halo_wide_eligible(3, 3, 1, 1, 128, 4, 4, affine={"scale": None})


def test_halo_wide_smem_bytes():
    # layer2 stride 1: two 4 x 6x6 x 128 B halo boxes (18 KB each) and 18 weight slots
    assert F.halo_wide_smem_bytes(128, 4, 4, 1) == 2 * (18 * 1024 + 9 * 8192) + 256 + 1024 + 1024
    # layer2.0.conv1: one 4 x 9x9 x 128 B box (40.5 KB, rounded up to 41 KB) and 9 weight slots
    assert F.halo_wide_smem_bytes(64, 8, 8, 2) == 41 * 1024 + 9 * 8192 + 256 + 1024 + 1024
    assert F.halo_wide_smem_bytes(128, 4, 4, 1) <= 227 * 1024
    for h in (2, 4, 8):
        assert F.halo_wide_smem_bytes(128, h, h, 1) <= 227 * 1024
    # 64 images of 1x1 need 2 x 72 KB of halo beside the 144 KB of weights
    assert F.halo_wide_smem_bytes(128, 1, 1, 1) > 227 * 1024 and not F.halo_wide_eligible(3, 3, 1, 1, 128, 1, 1)
    assert F.halo_wide_smem_bytes(256, 2, 2, 1) > 227 * 1024


def test_forced_halo_path_on_a_shape_no_halo_kernel_takes_is_refused():
    with pytest.raises(ValueError):
        F._conv_path("halo", F.halo_eligible(3, 3, 2, 1, 128, 4, 4) or F.halo_wide_eligible(3, 3, 2, 1, 128, 4, 4))
