"""Random-crop and horizontal-flip augmentation of NHWC image shards, drawn per sample and per epoch.

One definition, shared by every trainer.  The sample at position ``s`` of an epoch's gathered order (``0 .. n-1``, the
order the epoch's permutation puts the samples in) draws from ONE Philox4x32-10 output::

    x = philox4x32_10(counter = (s, epoch, stream_lo, stream_hi), key = (key_lo, key_hi))
    oy = x[0] % (2p + 1)      ox = x[1] % (2p + 1)      (0 when the kind has no crop)
    flip = x[2] & 1           (0 when the kind has no flip)
    out[s, h, w, c] = src[perm[s], h + oy - p, w' + ox - p, c]   if inside the image, else 0
    where w' = W - 1 - w when flip, else w

which is torchvision's ``RandomCrop(padding=p, fill=0)`` followed by ``RandomHorizontalFlip(0.5)``.  The CUDA trainer
computes it inside the epoch's batch gather (``F.gather_augment``, ``csrc/elementwise.cu``); the CPU trainers call
:func:`gather_augment_reference`, the torch form of the same formula.

The key and stream: :class:`~baton_b200.parallel.engine.FederatedEngine` derives the key from its ``seed`` (the same on
every rank) and uses ``stream = (round_index << 32) | client_id``.  A trainer used on its own draws a random key once
(or derives it from an explicit ``augment_seed``) and uses its run counter as the stream.
"""
from __future__ import annotations

import secrets
from dataclasses import dataclass
from typing import Optional, Tuple

import numpy as np
import torch

from ..parallel.dp import philox4x32_10

KINDS = {"crop": (True, False), "flip": (False, True), "crop_flip": (True, True)}
_M32, _M64 = 0xFFFFFFFF, 0xFFFFFFFFFFFFFFFF


@dataclass(frozen=True)
class AugmentConfig:
    """A normalized augmentation: ``padding`` is 0 for a kind without crop."""
    kind: str
    padding: int

    @property
    def crop(self) -> bool:
        return KINDS[self.kind][0]

    @property
    def flip(self) -> bool:
        return KINDS[self.kind][1]


def check_augment(kind: Optional[str], padding: int = 4) -> Optional[AugmentConfig]:
    """The normalized config of ``(kind, padding)``, or None for ``None`` / ``"none"``; ``ValueError`` for an unknown
    kind or a crop with ``padding < 1``."""
    if kind is None or kind == "none":
        return None
    if kind not in KINDS:
        raise ValueError("augment must be one of none, {}; got {!r}".format(", ".join(KINDS), kind))
    try:
        p = int(padding)
    except (TypeError, ValueError):
        raise ValueError("augment_padding must be an integer, got {!r}".format(padding)) from None
    if p != padding:
        raise ValueError("augment_padding must be an integer, got {!r}".format(padding))
    if not KINDS[kind][0]:
        return AugmentConfig(kind, 0)
    if p < 1:
        raise ValueError("a random crop needs augment_padding >= 1, got {!r}".format(padding))
    return AugmentConfig(kind, p)


def check_shard(cfg: AugmentConfig, X: torch.Tensor) -> None:
    """``ValueError`` unless ``X`` is an NHWC float image shard the crop fits: 4-D, bf16 / fp16 / fp32, with
    ``padding < H`` and ``padding < W``."""
    if X.dim() != 4 or X.dtype not in (torch.bfloat16, torch.float16, torch.float32):
        raise ValueError("augmentation needs NHWC image shards (4-D bf16 / fp16 / fp32), got {} {}".format(
            tuple(X.shape), X.dtype))
    H, W = X.shape[1], X.shape[2]
    if cfg.padding >= H or cfg.padding >= W:
        raise ValueError("augment_padding {} must be smaller than the image ({}x{})".format(cfg.padding, H, W))


def augment_key(seed: int) -> int:
    """The 64-bit Philox key of an augmentation seed (SplitMix64 of the seed, so nearby seeds give unrelated keys)."""
    z = (int(seed) + 0x9E3779B97F4A7C15) & _M64
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & _M64
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & _M64
    return z ^ (z >> 31)


def augment_draws(key: int, stream: int, epoch: int, positions, padding: int, flip: bool,
                  crop: bool = True) -> Tuple[np.ndarray, np.ndarray, np.ndarray]:
    """``(oy, ox, flip)`` int64 arrays of the given epoch positions; ``oy = ox = 0`` for ``padding = 0`` or no crop."""
    pos = np.asarray(positions, dtype=np.uint64).reshape(-1)
    ctr = np.stack([pos & np.uint64(_M32), np.full_like(pos, int(epoch) & _M32),
                    np.full_like(pos, int(stream) & _M32), np.full_like(pos, (int(stream) >> 32) & _M32)], axis=-1)
    key = int(key) & _M64
    x = philox4x32_10(ctr, (key & _M32, key >> 32)).astype(np.int64)
    span = 2 * int(padding) + 1 if crop else 1
    fl = (x[:, 2] & 1) if flip else np.zeros(len(pos), dtype=np.int64)
    return x[:, 0] % span, x[:, 1] % span, fl


def epoch_words(stream: int, n_epoch: int) -> torch.Tensor:
    """int32 ``[n_epoch, 3]`` host table of the kernel's per-epoch words ``{epoch, stream_lo, stream_hi}``."""
    lo, hi = int(stream) & _M32, (int(stream) >> 32) & _M32
    rows = [[e, lo, hi] for e in range(n_epoch)]
    return torch.tensor(np.array(rows, dtype=np.uint32).reshape(n_epoch, 3).view(np.int32))


def gather_augment_reference(X: torch.Tensor, idx: torch.Tensor, key: int, stream: int, epoch: int, padding: int,
                             crop: bool = True, flip: bool = True, s0: int = 0) -> torch.Tensor:
    """``augment(X[idx])`` in torch for output positions ``s0 .. s0 + len(idx) - 1``: pure data movement, so equal bit
    for bit to ``F.gather_augment`` on the same inputs."""
    n = idx.numel()
    H, W = X.shape[1], X.shape[2]
    p = int(padding) if crop else 0
    oy, ox, fl = (torch.from_numpy(a).to(X.device)
                  for a in augment_draws(key, stream, epoch, np.arange(s0, s0 + n), p, flip, crop))
    xp = torch.nn.functional.pad(X[idx.to(X.device)], (0, 0, p, p, p, p))      # zero fill around H and W
    ar_h = torch.arange(H, device=X.device)
    ar_w = torch.arange(W, device=X.device)
    cols = torch.where(fl.bool()[:, None], W - 1 - ar_w[None, :], ar_w[None, :]) + ox[:, None]
    rows = oy[:, None] + ar_h[None, :]
    return xp[torch.arange(n, device=X.device)[:, None, None], rows[:, :, None], cols[:, None, :]]


class AugmentStreams:
    """Key and stream of a trainer used on its own: ``augment_seed=None`` uses a random 64-bit key drawn once per
    trainer, an explicit seed :func:`augment_key` of it; the stream is the number of augmenting runs before this one
    unless the caller passes ``augment_stream``."""

    def __init__(self):
        self.key: Optional[int] = None
        self.runs = 0

    def next(self, augment_seed: Optional[int], augment_stream: Optional[int]) -> Tuple[int, int]:
        run = self.runs
        self.runs += 1
        if augment_seed is None:
            if self.key is None:
                self.key = secrets.randbits(64)
            key = self.key
        else:
            key = augment_key(augment_seed)
        return key, (run if augment_stream is None else int(augment_stream) & _M64)
