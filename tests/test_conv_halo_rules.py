"""CPU checks of the halo-kernel dispatch rule (layer1 and layer2 of ResNet-18 on 32x32 inputs) and of the in-graph
timeline's stamp pairing."""
import pytest

from baton_b200.ops import functional as F
from baton_b200.utils import trace

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


def test_flagship_shapes_select_exactly_the_layer1_and_layer2_gemms():
    fwd = [name for name, cin, _, k, s, p, h in RESNET18_32 if F.halo_eligible(k, k, s, p, cin, h, h)]
    # the input gradient gathers dy (Cout channels) over the input image; the stem's is never computed
    dgrad = [name for name, _, cout, k, s, p, h in RESNET18_32[1:]
             if F.halo_eligible(k, k, s, p, cout, h, h, dgrad=True)]
    layer1 = ["layer1.{}.conv{}".format(b, c) for b in range(2) for c in (1, 2)]
    layer2_s1 = ["layer2.0.conv2", "layer2.1.conv1", "layer2.1.conv2"]
    assert fwd == layer1 + ["layer2.0.conv1"] + layer2_s1
    assert dgrad == layer1 + layer2_s1


# args: (kh, kw, stride, pad, gathered channels, h, w[, affine, dgrad])
@pytest.mark.parametrize("args,ok", [
    # around the stride-1 64-channel form
    ((3, 3, 1, 1, 64, 8, 8), True),
    ((3, 3, 1, 1, 64, 4, 4), True),
    ((3, 3, 1, 1, 64, 1, 1), True),
    ((3, 3, 1, 1, 64, 4, 8), True),
    ((3, 3, 1, 1, 128, 8, 8), True),                 # two channel blocks: the stride-1 128-channel form
    ((3, 3, 2, 1, 64, 8, 8), True),                  # stride 2: the stride-2 64-channel form
    ((3, 3, 1, 0, 64, 8, 8), False),                 # not "same"
    ((1, 1, 1, 0, 64, 8, 8), False),
    ((3, 3, 1, 1, 64, 8, 16), False),                # 128 pixels: a 64-row tile holds no whole image
    ((3, 3, 1, 1, 64, 6, 6), False),                 # 64 % 36 != 0
    # around the stride-1 128-channel and stride-2 64-channel forms
    ((3, 3, 1, 1, 128, 4, 4), True),
    ((3, 3, 1, 1, 128, 4, 4, None, True), True),
    ((3, 3, 2, 1, 64, 8, 8), True),
    ((3, 3, 2, 1, 64, 8, 8, None, True), False),     # stride-2 input gradients have their own kernel
    ((3, 3, 1, 1, 128, 2, 2), True),
    ((3, 3, 1, 1, 128, 8, 8), True),
    ((3, 3, 2, 1, 64, 4, 4), True),                  # 2x2 outputs, 16 images per tile
    ((3, 3, 2, 1, 64, 16, 16), True),                # one 8x8 output image per tile
    ((3, 3, 1, 1, 64, 8, 8), True),                  # one channel block: the stride-1 64-channel form
    ((3, 3, 1, 1, 256, 2, 2), False),                # four channel blocks: 36 k-tiles do not fit
    ((3, 3, 2, 1, 128, 4, 4), False),
    ((3, 3, 1, 0, 128, 4, 4), False),
    ((1, 1, 1, 0, 128, 4, 4), False),
    ((3, 3, 1, 1, 128, 6, 6), False),                # 64 % 36 != 0
    ((3, 3, 2, 1, 64, 32, 32), False),               # 256 output pixels: a 64-row tile holds no whole image
])
def test_halo_rule(args, ok):
    assert F.halo_eligible(*args) is ok


def test_halo_rule_declines_the_affine_epilogue():
    for args in ((3, 3, 1, 1, 64, 8, 8), (3, 3, 1, 1, 128, 4, 4), (3, 3, 2, 1, 64, 8, 8)):
        assert not F.halo_eligible(*args, affine={"scale": None}), args


def test_halo_smem_fits_every_eligible_size():
    assert F.halo_smem_bytes(8, 8) == 13 * 1024 + 9 * 8192 + 128 + 1024 + 1024
    for h, w in ((1, 1), (1, 2), (2, 2), (4, 4), (8, 8), (4, 16), (1, 64)):
        assert F.halo_smem_bytes(h, w) <= 227 * 1024


def test_halo_smem_bytes_of_the_layer2_forms():
    # layer2 stride 1: two 4 x 6x6 x 128 B halo boxes (18 KB each), 18 weight slots and 19 mbarriers (256 B)
    assert F.halo_smem_bytes(4, 4, c=128) == 2 * (18 * 1024 + 9 * 8192) + 256 + 1024 + 1024
    # layer2.0.conv1: one 4 x 9x9 x 128 B box (40.5 KB, rounded up to 41 KB), 9 weight slots and 10 mbarriers (128 B)
    assert F.halo_smem_bytes(8, 8, c=64, stride=2) == 41 * 1024 + 9 * 8192 + 128 + 1024 + 1024
    assert F.halo_smem_bytes(4, 4, c=128) <= 227 * 1024
    for h in (2, 4, 8):
        assert F.halo_smem_bytes(h, h, c=128) <= 227 * 1024
    # 64 images of 1x1 need 2 x 72 KB of halo beside the 144 KB of weights
    assert F.halo_smem_bytes(1, 1, c=128) > 227 * 1024 and not F.halo_eligible(3, 3, 1, 1, 128, 1, 1)
    assert F.halo_smem_bytes(2, 2, c=256) > 227 * 1024


@pytest.mark.parametrize("rows,mc", [(8192, 4), (64 * 62, 2), (8064, 2), (64 * 63, 1), (192, 1), (64, 1)])
def test_halo_cluster(rows, mc):
    assert F.halo_cluster(rows) == mc


def test_forced_path_is_checked():
    with pytest.raises(ValueError):
        F._conv_path("halo", False)
    with pytest.raises(ValueError):
        F._conv_path("fast", True)
    assert F._conv_path(None, True) == "halo" and F._conv_path(None, False) == "im2col"
    assert F._conv_path("im2col", True) == "im2col"


def test_forced_halo_path_on_a_shape_no_halo_kernel_takes_is_refused():
    with pytest.raises(ValueError):
        F._conv_path("halo", F.halo_eligible(3, 3, 2, 1, 128, 4, 4))


def test_timeline_pairs_resident_and_deps_stamps_per_kernel():
    # tags: tu * 100000 + line; the resident stamp (negative) and the deps-done stamp of one kernel differ in line
    names = {101: "gemm", 105: "gemm", 201: "bn", 207: "bn"}
    rec = [(0, -101), (10, 105),      # gemm resident at 0, deps done at 10
           (4, -201),                  # bn resident while gemm runs (PDL overlap)
           (30, 207),                  # bn deps done
           (12, -101), (40, 105),      # second gemm
           (trace.POINT_BASE + 3, trace.POINT_BASE + 105)]   # intra-kernel point: ignored
    rec.sort()
    rows = trace.timeline_rows(rec, name=lambda t: names[abs(t)])
    assert [r["name"] for r in rows] == ["gemm", "bn", "gemm"]
    assert [r["early_ns"] for r in rows] == [10, 26, 28]
    assert [r["slot_ns"] for r in rows] == [20, 10, 0]


def test_timeline_without_resident_stamp_has_no_overlap():
    rows = trace.timeline_rows([(5, 105)], name=lambda t: "gemm")
    assert rows[0]["early_ns"] == 0 and rows[0]["slot_ns"] == 0
