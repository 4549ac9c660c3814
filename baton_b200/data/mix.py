"""Mixup, CutMix and label smoothing of local training: one lambda per batch, the batch rolled by one as the partner.

One definition, shared by every trainer, following torchvision v2's ``MixUp`` / ``CutMix``:

* **Partner.**  Within each batch of ``L`` rows (epoch positions ``b*B .. b*B + L - 1``; the ragged last batch rolls
  within itself), row ``j`` is mixed with row ``(j - 1 + L) % L`` -- ``batch.roll(1, 0)``.
* **Order.**  Each row is first cropped / flipped with its own draws (``data/augment.py``); the two augmented images are
  then mixed.
* **Draws.**  One row per ``(epoch, batch)`` from :func:`mix_table`: a ``numpy.random.Generator(Philox)`` seeded only
  from the augmentation key, the stream and the epoch draws per batch, in this order, ``u = random()`` (``mixup_cutmix``
  only: CutMix iff ``u < 0.5``), ``lam = beta(alpha, alpha)`` and, for CutMix, ``cy = floor(H random())`` and
  ``cx = floor(W random())`` (uniform on ``0 .. H-1`` and ``0 .. W-1``).
* **Mixup.**  ``out = round_dtype(fp32(fp32(a * lam) + fp32(b * lam1)))``, each product and the sum rounded on its own.
* **CutMix.**  ``r = 0.5 sqrt(1 - lam)``, ``hh = int(r H)``, ``hw = int(r W)``, box ``y0 = max(cy - hh, 0)``,
  ``y1 = min(cy + hh, H)`` (same for x); pixels inside come from the partner and the label weight becomes
  ``lam = 1 - (y1 - y0)(x1 - x0) / (H W)``.
* **Soft target** of row ``j`` with own label ``a`` and partner label ``b``:
  ``q = (1 - eps)(lam 1[a] + lam1 1[b]) + eps / C``; loss ``logsumexp(z) - sum_c q_c z_c`` = ``lam CE(z, a, eps) +
  lam1 CE(z, b, eps)``; gradient ``softmax(z) - q``.  Without mixing ``lam = 1`` and ``b = a``: label smoothing.  The
  training "correct" count is ``lam [argmax = a] + lam1 [argmax = b]``.

A mix row is 8 int32 words: ``lam`` and ``lam1 = 1 - lam`` (computed in float64, stored as fp32 bit patterns), the kind
(``MIXUP`` / ``CUTMIX``) and the box ``y0, y1, x0, x1`` (empty for mixup).  The CUDA trainer mixes inside the
epoch's batch gather (``F.gather_augment(mix_rows=...)``) and applies the soft target in the fused loss kernels; the
CPU trainers call :func:`mix_batch_reference` and :func:`soft_cross_entropy`.  Evaluation always uses hard labels.
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import NamedTuple, Optional

import numpy as np
import torch

KINDS = ("mixup", "cutmix", "mixup_cutmix")
MIX_ROW = 8
MIXUP, CUTMIX = 0, 1
_M32, _M64 = 0xFFFFFFFF, 0xFFFFFFFFFFFFFFFF


@dataclass(frozen=True)
class MixConfig:
    """``kind`` None: label smoothing only (no mixing, no draws)."""
    kind: Optional[str]
    alpha: float
    smoothing: float


def check_mix(kind: Optional[str], alpha: float = 1.0, label_smoothing: float = 0.0) -> Optional[MixConfig]:
    """The normalized config, or None when neither mixing nor label smoothing is on; ``ValueError`` for an unknown kind,
    an ``alpha`` that is not a finite number > 0, or ``label_smoothing`` outside [0, 1)."""
    if kind == "none":
        kind = None
    if kind is not None and kind not in KINDS:
        raise ValueError("mix must be one of none, {}; got {!r}".format(", ".join(KINDS), kind))
    try:
        a, eps = float(alpha), float(label_smoothing)
    except (TypeError, ValueError):
        raise ValueError("mix_alpha and label_smoothing must be numbers, got {!r}, {!r}".format(
            alpha, label_smoothing)) from None
    if not 0.0 < a < math.inf:
        raise ValueError("mix_alpha must be a finite number > 0, got {!r}".format(alpha))
    if not 0.0 <= eps < 1.0:
        raise ValueError("label_smoothing must be in [0, 1), got {!r}".format(label_smoothing))
    if kind is None and eps == 0.0:
        return None
    return MixConfig(kind, a, eps)


def check_mix_loss(cfg: Optional[MixConfig], loss) -> None:
    """``ValueError`` unless a run with ``cfg`` trains with the cross-entropy loss (soft targets need one)."""
    if cfg is not None and (callable(loss) or loss not in ("ce", "cross_entropy")):
        raise ValueError("mix and label_smoothing need the cross-entropy loss, got loss={!r}".format(loss))


def check_mix_shard(cfg: Optional[MixConfig], X: torch.Tensor) -> None:
    """``ValueError`` when ``cfg`` mixes and ``X`` is not an NHWC float image shard (token, MLP and linear inputs)."""
    if cfg is None or cfg.kind is None:
        return
    if X.dim() != 4 or X.dtype not in (torch.bfloat16, torch.float16, torch.float32):
        raise ValueError("mix needs NHWC image shards (4-D bf16 / fp16 / fp32), got {} {}".format(
            tuple(X.shape), X.dtype))


def mix_generator(key: int, stream: int, epoch: int) -> np.random.Generator:
    """The generator of one epoch's mix rows: Philox seeded from ``(key, stream, epoch)`` only."""
    key, stream = int(key) & _M64, int(stream) & _M64
    seq = np.random.SeedSequence([key & _M32, key >> 32, stream & _M32, stream >> 32, int(epoch) & _M32])
    return np.random.Generator(np.random.Philox(seq))


def mix_table(key: int, stream: int, epoch: int, n_batches: int, cfg: MixConfig, H: int, W: int) -> np.ndarray:
    """int32 ``[n_batches, MIX_ROW]`` mix rows of one epoch (module docstring); row ``b`` does not depend on
    ``n_batches`` beyond ``b``."""
    g = mix_generator(key, stream, epoch)
    out = np.zeros((n_batches, MIX_ROW), dtype=np.int32)
    if cfg.kind == "mixup":
        lam = g.beta(cfg.alpha, cfg.alpha, n_batches)        # the same draws as one call per batch
    else:
        lam = np.empty(n_batches)
        for b in range(n_batches):
            cut = cfg.kind == "cutmix" or g.random() < 0.5
            lam[b] = g.beta(cfg.alpha, cfg.alpha)
            if cut:
                cy, cx = int(H * g.random()), int(W * g.random())
                r = 0.5 * math.sqrt(1.0 - lam[b])
                hh, hw = int(r * H), int(r * W)
                y0, y1, x0, x1 = max(cy - hh, 0), min(cy + hh, H), max(cx - hw, 0), min(cx + hw, W)
                out[b, 2:7] = (CUTMIX, y0, y1, x0, x1)
                lam[b] = 1.0 - (y1 - y0) * (x1 - x0) / (H * W)
    out[:, 0] = lam.astype(np.float32).view(np.int32)
    out[:, 1] = (1.0 - lam).astype(np.float32).view(np.int32)
    return out


def mix_rows(key: int, stream: int, n_epoch: int, n_batches: int, cfg: MixConfig, H: int, W: int) -> torch.Tensor:
    """int32 ``[n_epoch, n_batches, MIX_ROW]`` host table of a run: :func:`mix_table` of every epoch."""
    return torch.from_numpy(np.stack([mix_table(key, stream, e, n_batches, cfg, H, W) for e in range(n_epoch)]))


class Row(NamedTuple):
    lam: float
    lam1: float
    kind: int
    y0: int
    y1: int
    x0: int
    x1: int


def decode_row(row) -> Row:
    """The fields of one mix row (any int32 sequence of ``MIX_ROW`` words)."""
    w = np.asarray(torch.as_tensor(row).cpu(), dtype=np.int32).reshape(-1)
    lam, lam1 = w[:2].view(np.float32)
    return Row(float(lam), float(lam1), int(w[2]), int(w[3]), int(w[4]), int(w[5]), int(w[6]))


class SoftTarget(NamedTuple):
    """Row ``j``'s target: ``(1 - eps)(lam 1[a_j] + lam1 1[b_j]) + eps / C``."""
    a: torch.Tensor
    b: torch.Tensor
    lam: float
    lam1: float
    eps: float


def mix_batch_reference(batch: torch.Tensor, labels: torch.Tensor, row, eps: float = 0.0):
    """``(mixed batch, SoftTarget)`` of one batch (already cropped / flipped: ``gather_augment_reference``'s output)
    under the mix row ``row`` (None: no mixing, label smoothing ``eps`` only).  Equal bit for bit to the mixing
    gather."""
    if row is None:
        return batch, SoftTarget(labels, labels, 1.0, 0.0, float(eps))
    r = decode_row(row)
    partner = batch.roll(1, 0)
    if r.kind == CUTMIX:
        out = batch.clone()
        out[:, r.y0:r.y1, r.x0:r.x1] = partner[:, r.y0:r.y1, r.x0:r.x1]
    else:
        lam = torch.tensor(r.lam, dtype=torch.float32)
        lam1 = torch.tensor(r.lam1, dtype=torch.float32)
        out = ((batch.float() * lam) + (partner.float() * lam1)).to(batch.dtype)
    return out, SoftTarget(labels, labels.roll(1, 0), r.lam, r.lam1, float(eps))


def soft_cross_entropy(logits: torch.Tensor, t: SoftTarget) -> torch.Tensor:
    """Batch-mean loss of the soft target: ``lam CE(z, a, eps) + lam1 CE(z, b, eps)`` in torch."""
    z = logits.float()
    loss = t.lam * torch.nn.functional.cross_entropy(z, t.a, label_smoothing=t.eps)
    if t.lam1 != 0.0:
        loss = loss + t.lam1 * torch.nn.functional.cross_entropy(z, t.b, label_smoothing=t.eps)
    return loss


def soft_hits(logits: torch.Tensor, t: SoftTarget) -> torch.Tensor:
    """The training "correct" count ``sum_j lam [argmax_j = a_j] + lam1 [argmax_j = b_j]``."""
    am = logits.argmax(-1)
    return t.lam * (am == t.a).sum().float() + t.lam1 * (am == t.b).sum().float()
