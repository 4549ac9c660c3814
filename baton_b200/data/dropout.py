"""Dropout of BERT training, drawn from a counter so every trainer and every kernel draws the same masks.

One definition, shared by every trainer.  A BERT model with ``L`` layers has ``2 + 3L`` dropout sites, Hugging-Face
``BertForSequenceClassification``'s positions:

    site 0        [B*S, D]     output of the embeddings LayerNorm                      (hidden_dropout_prob)
    site 1 + 3l   [B, H, S, S] attention probabilities of layer l, before P V         (attention_probs_dropout_prob)
    site 2 + 3l   [B*S, D]     output of attn_out of layer l, before the residual add  (hidden_dropout_prob)
    site 3 + 3l   [B*S, D]     output of ffn_out of layer l, before the residual add   (hidden_dropout_prob)
    site 1 + 3L   [B, D]       the pooled vector, before the classifier                (classifier_dropout)

Element ``i`` of a site is its flat row-major index in the tensor above (for the probabilities, the index into the
``[B*H*S, S]`` probability buffer).  It draws word ``i & 3`` of ONE Philox4x32-10 output::

    x = philox4x32_10(counter = (i >> 2, 0x80000000 | site << 22 | t, stream_lo, stream_hi), key = (key_lo, key_hi))

where ``t = epoch * steps_per_epoch + step`` is the local step of the run (a ragged last batch is a step).  The element
is kept iff ``x[i & 3] >= T`` with ``T = floor(p * 2^32)`` (fp64 on the host); a kept value is multiplied by
``s = fp32(1 / (1 - p))`` in fp32, before any bf16 rounding, and a dropped one becomes 0.  Nine bits of site and 22 of
step: a run with more is a ``ValueError``.  The top bit of word 1 keeps these counters apart from augmentation's
``(s, epoch, stream_lo, stream_hi)``, whose epoch is below 2^31.

The key and stream are augmentation's (``data/augment.py``): :class:`~baton_b200.parallel.engine.FederatedEngine` uses
the key of its ``seed`` and ``stream = (round_index << 32) | client_id``; a trainer used on its own uses
``AugmentStreams`` with ``augment_seed`` / ``augment_stream``.  Nothing is dropped in eval mode, and a model whose
probabilities are all 0 runs exactly the kernels it runs without dropout.  The CUDA modules draw the masks inside the
fused attention, LayerNorm and softmax kernels (``csrc/dropout.cuh``); the CPU modules call :func:`dropout_reference`.
"""
from __future__ import annotations

import math
from typing import Optional

import numpy as np
import torch

from ..parallel.dp import philox4x32_10

SITE_BITS, STEP_BITS = 9, 22
MAX_SITES, MAX_STEPS = 1 << SITE_BITS, 1 << STEP_BITS
_M32 = 0xFFFFFFFF


def check_dropout(p, name: str = "dropout") -> float:
    """``p`` as a float; ``ValueError`` unless it is a number in ``[0, 1)``."""
    try:
        v = float(p)
    except (TypeError, ValueError):
        raise ValueError("{} must be a probability in [0, 1), got {!r}".format(name, p)) from None
    if isinstance(p, bool) or not (0.0 <= v < 1.0):
        raise ValueError("{} must be a probability in [0, 1), got {!r}".format(name, p))
    return v


def threshold(p: float) -> int:
    """``T = floor(p * 2^32)``: an element is kept iff its word is ``>= T``."""
    return int(math.floor(float(p) * 4294967296.0))


def scale(p: float) -> float:
    """``s = fp32(1 / (1 - p))`` (as a Python float holding that fp32 value)."""
    return float(np.float32(1.0 / (1.0 - float(p))))


def counter_word(site: int, t: int) -> int:
    """Word 1 of the counter, ``0x80000000 | site << 22 | t``; ``ValueError`` outside 9 bits of site and 22 of step."""
    if not (0 <= int(site) < MAX_SITES):
        raise ValueError("dropout site {} needs more than {} bits".format(site, SITE_BITS))
    if not (0 <= int(t) < MAX_STEPS):
        raise ValueError("dropout step {} needs more than {} bits".format(t, STEP_BITS))
    return 0x80000000 | (int(site) << STEP_BITS) | int(t)


def check_run(n_sites: int, n_steps: int) -> None:
    """``ValueError`` when a run of ``n_steps`` local steps over ``n_sites`` sites does not fit the counter."""
    if n_sites > MAX_SITES:
        raise ValueError("dropout supports at most {} sites, the model has {}".format(MAX_SITES, n_sites))
    if n_steps > MAX_STEPS:
        raise ValueError("dropout supports at most 2^{} local steps per run, got {}".format(STEP_BITS, n_steps))


def dropout_keep(key: int, stream: int, site: int, t: int, n: int, p: float) -> np.ndarray:
    """bool ``[n]``: which elements ``0 .. n-1`` of the site are kept at local step ``t``."""
    w1 = counter_word(site, t)
    nq = (int(n) + 3) // 4
    if nq > 1 << 32:
        raise ValueError("a dropout site holds at most 2^34 elements")
    q = np.arange(nq, dtype=np.uint64)
    ctr = np.stack([q, np.full_like(q, w1), np.full_like(q, int(stream) & _M32),
                    np.full_like(q, (int(stream) >> 32) & _M32)], axis=-1)
    key = int(key) & 0xFFFFFFFFFFFFFFFF
    x = philox4x32_10(ctr, (key & _M32, key >> 32)).reshape(-1)[: int(n)]
    return x >= np.uint32(threshold(p))


def dropout_reference(x: torch.Tensor, key: int, stream: int, site: int, t: int, p: float) -> torch.Tensor:
    """``x`` with the site's mask applied: kept elements times ``s`` (in ``x``'s dtype, fp32 for fp32), dropped ones 0."""
    keep = torch.from_numpy(dropout_keep(key, stream, site, t, x.numel(), p)).to(x.device).view(x.shape)
    return torch.where(keep, x * torch.tensor(scale(p), dtype=x.dtype, device=x.device), torch.zeros_like(x))


class DropoutRun:
    """The state a model's dropout sites read during one training step: the key and stream of the run, and the epoch
    and step.  A trainer calls :meth:`begin` before a run, :meth:`at` before every step and :meth:`end` after; the sites
    are inert outside a run (and in eval mode).  ``words`` is the device int32 ``{epoch, stream_lo, stream_hi}`` the
    CUDA kernels read -- a captured epoch graph's word buffer, rewritten before each replay."""

    def __init__(self):
        self.key: Optional[int] = None
        self.stream = 0
        self.epoch = 0
        self.step = 0
        self.steps = 1
        self.words: Optional[torch.Tensor] = None

    @property
    def active(self) -> bool:
        return self.key is not None

    def begin(self, key: int, stream: int, steps: int, n_epoch: int, n_sites: int) -> None:
        check_run(n_sites, int(steps) * int(n_epoch))
        self.key, self.stream, self.steps = int(key), int(stream), int(steps)
        self.epoch = self.step = 0

    def at(self, epoch: int, step: int, words: Optional[torch.Tensor] = None) -> None:
        self.epoch, self.step = int(epoch), int(step)
        if words is not None:
            self.words = words

    def end(self) -> None:
        self.key = None
        self.words = None

    @property
    def t(self) -> int:
        return self.epoch * self.steps + self.step

    def kernel_args(self, site: int, p: float) -> tuple:
        """The trailing arguments of a dropout kernel entry point for ``site`` at the current step."""
        k = self.key & 0xFFFFFFFFFFFFFFFF
        return (self.words, k - (1 << 64) if k >> 63 else k, int(site), self.step, self.steps, threshold(p), scale(p))

    def apply(self, x: torch.Tensor, site: int, p: float) -> torch.Tensor:
        """:func:`dropout_reference` of ``x`` at the current step (the CPU form of every site)."""
        return dropout_reference(x, self.key, self.stream, site, self.t, p)
