"""Stride-2 implicit-GEMM input gradient (sub-pixel decomposition into four parity classes of dx pixels) against the
explicit ``F.gemm(dy, W, b_mn=True)`` + ``F.col2im`` lowering, and the per-class tap tables it runs from."""
from collections import Counter

import pytest
import torch

from baton_b200.ops import functional as F

BF16 = torch.bfloat16


def _rel(a, b):
    a, b = a.float(), b.float()
    return float((a - b).abs().max() / (b.abs().max() + 1e-6))


@pytest.mark.parametrize("k,pad", [(3, 1), (1, 0)])
@pytest.mark.parametrize("h,w", [(8, 8), (4, 4), (2, 2), (1, 1), (7, 7), (5, 9), (6, 3)])
def test_s2_tap_tables_cover_every_contribution_once(k, pad, h, w):
    ho, wo = F.conv_out_size(h, k, 2, pad), F.conv_out_size(w, k, 2, pad)
    # every (dx pixel, tap, dy pixel) term of the stride-2 convolution's input gradient
    want = Counter()
    for p in range(ho):
        for q in range(wo):
            for r in range(k):
                for s in range(k):
                    y, x = 2 * p - pad + r, 2 * q - pad + s
                    if 0 <= y < h and 0 <= x < w:
                        want[(y, x, r * k + s, p, q)] += 1
    classes = F.conv_s2_dgrad_taps(k, k, pad, ho, wo)
    assert classes is not None and len(classes) == 4
    got = Counter()
    for c, taps in enumerate(classes):
        a, b = c >> 1, c & 1
        assert len(taps) <= F.S2_MAX_TAPS
        for i in range(ho):              # the kernel enumerates the dy grid for every class
            for j in range(wo):
                y, x = 2 * i + a, 2 * j + b
                if y >= h or x >= w:
                    continue
                for t, dp, dq in taps:
                    assert dp >= 0 and dq >= 0
                    if i + dp < ho and j + dq < wo:      # outside dy: the gather reads zero
                        r, s = divmod(t, k)
                        assert 2 * (i + dp) - pad + r == y and 2 * (j + dq) - pad + s == x
                        got[(y, x, t, i + dp, j + dq)] += 1
    assert got == want
    # the kernel's grid must reach every dx pixel
    assert (h + 1) // 2 <= ho and (w + 1) // 2 <= wo


def test_s2_tap_tables_decline_negative_offsets():
    assert F.conv_s2_dgrad_taps(7, 7, 3, 16, 16) is None      # 7x7 pad 3: some taps would need dy[i - 1]


# ResNet-18 stride-2 convolutions at batch 128 (32x32 inputs), odd sizes at batch 3, and a long K (32 k tiles) over few tiles
S2_SHAPES = [
    (128, 64, 128, 3, 1, 8, 8), (128, 64, 128, 1, 0, 8, 8),          # layer2.0 conv1 / downsample
    (128, 128, 256, 3, 1, 4, 4), (128, 128, 256, 1, 0, 4, 4),        # layer3.0
    (128, 256, 512, 3, 1, 2, 2), (128, 256, 512, 1, 0, 2, 2),        # layer4.0 (1x1 output)
    (3, 64, 64, 3, 1, 7, 7), (3, 64, 128, 3, 1, 5, 9), (3, 128, 64, 1, 0, 5, 9),
    (8, 64, 512, 3, 1, 8, 8),
]


@pytest.mark.gpu
@pytest.mark.parametrize("n,cin,cout,k,pad,h,w", S2_SHAPES)
def test_s2_implicit_dgrad_matches_gemm_col2im(n, cin, cout, k, pad, h, w):
    dev = torch.device("cuda:0")
    torch.manual_seed(n + cin + cout + k + h + w)
    ho, wo = F.conv_out_size(h, k, 2, pad), F.conv_out_size(w, k, 2, pad)
    dy = torch.randn(n, ho, wo, cout, device=dev).to(BF16)
    w2d = (torch.randn(cout, k * k * cin, device=dev) / (k * k * cin) ** 0.5).to(BF16)
    dx_ref = F.col2im(F.gemm(dy.view(-1, cout), w2d, b_mn=True), (n, h, w, cin), k, k, 2, pad, ho, wo)
    out = torch.full((n, h, w, cin), float("nan"), dtype=BF16, device=dev)     # every element must be written
    dx = F.conv_igemm_dgrad(dy, w2d, (n, h, w, cin), k, k, pad, stride=2, out=out)
    torch.cuda.synchronize()
    assert dx is not None and dx.data_ptr() == out.data_ptr()
    assert not torch.isnan(dx).any()
    assert _rel(dx, dx_ref) < 1e-2
    if k == 1:       # classes without taps: exact zeros
        assert torch.count_nonzero(dx[:, 1::2]) == 0 and torch.count_nonzero(dx[:, :, 1::2]) == 0
