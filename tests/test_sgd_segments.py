"""Chunk table of the leftover optimizer pass (``ops.functional.sgd_segments``): together with the blocks the
weight-gradient epilogues updated it must cover the parameter arena exactly once."""
import numpy as np
import pytest

from baton_b200.ops import functional as F


def _coverage(n, fused, segs):
    hits = np.zeros(n, dtype=np.int64)
    for off, rows, cols, ld in fused:
        for r in range(rows):
            hits[off + r * ld: off + r * ld + cols] += 1
    for off, length, _ in segs:
        hits[off: off + length] += 1
    return hits


def _check(n, fused, nograd, chunk):
    segs = F.sgd_segments(n, fused, nograd, chunk=chunk)
    assert (_coverage(n, fused, segs) == 1).all()
    offs = [s[0] for s in segs]
    assert offs == sorted(offs)
    ng = np.zeros(n, dtype=bool)
    for off, length in nograd:
        ng[off: off + length] = True
    for off, length, kind in segs:
        assert 0 < length <= chunk
        assert kind in (0, 1)
        assert ng[off: off + length].all() if kind == 1 else not ng[off: off + length].any()
    return segs


def test_resnet18_deep_layer_layout():
    # a 3x3 conv on a 1x1 map (centre tap only: rows of Cin at pitch 9 Cin) between fully fused igemm weights and
    # parameters that keep their gradient (BatchNorm, head)
    cin = cout = 512
    conv_a = (1024, 256, 2304, 2304)                 # igemm wgrad, [Cout, 9 Cin] contiguous
    centre_off = 1024 + 256 * 2304 + 64
    centre = (centre_off + 4 * cin, cout, cin, 9 * cin)
    n = centre_off + cout * 9 * cin + 5130
    segs = _check(n, [conv_a, centre], [(centre_off, cout * 9 * cin)], chunk=F.SGD_CHUNK)
    nograd = sum(length for _, length, kind in segs if kind == 1)
    assert nograd == cout * 8 * cin
    assert all(off % 4 == 0 for off, _, _ in segs)      # the kernel's 16-byte path


def test_nothing_fused_is_one_pass_over_the_arena():
    segs = _check(10_000, [], [], chunk=4096)
    assert [(s[0], s[1]) for s in segs] == [(0, 4096), (4096, 4096), (8192, 1808)]
    assert all(s[2] == 0 for s in segs)


@pytest.mark.parametrize("seed", range(5))
def test_random_layouts(seed):
    rng = np.random.default_rng(seed)
    n, pos, fused, nograd = 0, 0, [], []
    for _ in range(12):
        pos += int(rng.integers(0, 40)) * 8
        rows, cols = int(rng.integers(1, 9)), int(rng.integers(1, 6)) * 8
        if rng.random() < 0.4:                          # centre-tap-like: strided rows inside a no-grad parameter
            taps = int(rng.integers(2, 5))
            ld = taps * cols
            fused.append((pos + int(rng.integers(0, taps)) * cols, rows, cols, ld))
            nograd.append((pos, rows * ld))
            pos += rows * ld
        else:
            fused.append((pos, rows, cols, cols))
            pos += rows * cols
    n = pos + int(rng.integers(0, 100))
    _check(n, fused, nograd, chunk=int(rng.integers(1, 64)) * 8)


def test_overlapping_blocks_are_rejected():
    with pytest.raises(ValueError):
        F.sgd_segments(100, [(0, 1, 16, 16), (8, 1, 16, 16)], [])
    with pytest.raises(ValueError):
        F.sgd_segments(100, [(96, 1, 16, 16)], [])
