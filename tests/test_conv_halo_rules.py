"""CPU checks of the halo-kernel dispatch rule and of the in-graph timeline's stamp pairing."""
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


def test_flagship_shapes_select_exactly_the_layer1_gemms():
    fwd = [name for name, cin, _, k, s, p, h in RESNET18_32 if F.halo_eligible(k, k, s, p, cin, h, h)]
    # the input gradient gathers dy (Cout channels) over the input image; the stem's is never computed
    dgrad = [name for name, _, cout, k, s, p, h in RESNET18_32[1:] if F.halo_eligible(k, k, s, p, cout, h, h)]
    layer1 = ["layer1.{}.conv{}".format(b, c) for b in range(2) for c in (1, 2)]
    assert fwd == layer1 and dgrad == layer1


@pytest.mark.parametrize("args,ok", [
    ((3, 3, 1, 1, 64, 8, 8), True),
    ((3, 3, 1, 1, 64, 4, 4), True),
    ((3, 3, 1, 1, 64, 1, 1), True),
    ((3, 3, 1, 1, 64, 4, 8), True),
    ((3, 3, 1, 1, 128, 8, 8), False),     # two channel blocks
    ((3, 3, 2, 1, 64, 8, 8), False),      # stride 2
    ((3, 3, 1, 0, 64, 8, 8), False),      # not "same"
    ((1, 1, 1, 0, 64, 8, 8), False),
    ((3, 3, 1, 1, 64, 8, 16), False),     # 128 pixels: a 64-row tile holds no whole image
    ((3, 3, 1, 1, 64, 6, 6), False),      # 64 % 36 != 0
])
def test_halo_rule(args, ok):
    assert F.halo_eligible(*args) is ok


def test_halo_rule_declines_the_affine_epilogue():
    assert not F.halo_eligible(3, 3, 1, 1, 64, 8, 8, affine={"scale": None})


def test_halo_smem_fits_every_eligible_size():
    assert F.halo_smem_bytes(8, 8) == 13 * 1024 + 9 * 8192 + 128 + 1024 + 1024
    for h, w in ((1, 1), (1, 2), (2, 2), (4, 4), (8, 8), (4, 16), (1, 64)):
        assert F.halo_smem_bytes(h, w) <= 227 * 1024


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
