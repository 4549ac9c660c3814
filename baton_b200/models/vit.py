"""Vision Transformers for small images on the sm_90a layers, with torchvision's parameters.

``VisionTransformer`` computes torchvision's ``torchvision.models.vision_transformer.VisionTransformer(image_size,
patch_size, num_layers, num_heads, hidden_dim, mlp_dim, num_classes)`` and has its ``state_dict``: the same keys and
shapes, so checkpoints load both ways with ``strict=True`` and no mapping.  torchvision's packed ``in_proj_weight``
(rows q; k; v) is the packed ``qkv`` operand of ``ops.nn.attention``.

Forward on CUDA, for NHWC bf16 images ``[B, H, W, 3]``:
  1. the patch embedding is the ``ops.nn.Conv2d`` path (``K = 3 p^2``, without its bias);
  2. one token kernel builds ``[class token; patches + bias] + pos_embedding``, each token summed in fp32 and rounded
     once;
  3. every pre-LN block runs ``in_proj`` GEMM, the fused attention (``S = (H/p)^2 + 1 < 128``), ``out_proj``, the
     fused add + LayerNorm that also writes the residual sum, ``mlp.0`` with the exact (erf) GELU, ``mlp.3`` and the
     next fused add + LayerNorm (the next block's ``ln_1``, or ``encoder.ln`` after the last block);
  4. ``heads.head`` on the class-token rows, fp32 logits.

Layer 0's ``ln_1`` is a plain LayerNorm of the tokens.  Without dropout or stochastic depth (torchvision's defaults),
training and evaluation compute the same function.  On a CPU tensor every layer falls back to its ``torch`` form.
"""
from __future__ import annotations

import math
from collections import OrderedDict
from typing import Optional

import torch
from torch import nn

from ..ops import nn as bnn
from .base import FederatedModule

HEAD_DIM = 64        # the fused attention kernels' d_head
MAX_TOKENS = 128     # ... and their largest sequence


class _PatchEmbed(bnn.Conv2d):
    """torchvision's ``conv_proj``: a stride-``p`` ``p x p`` convolution with a bias.  The convolution runs without it;
    the token kernel adds the bias (``ops.nn.vit_tokens``)."""

    def __init__(self, hidden_dim: int, patch_size: int):
        super().__init__(3, hidden_dim, patch_size, patch_size, 0)
        self.bias = nn.Parameter(torch.zeros(hidden_dim))


class _SelfAttention(nn.Module):
    """``nn.MultiheadAttention(batch_first=True)`` self-attention under its ``state_dict`` names: ``in_proj_weight``
    ``[3D, D]``, ``in_proj_bias`` and ``out_proj``."""

    def __init__(self, hidden_dim: int, num_heads: int):
        super().__init__()
        self.num_heads = num_heads
        self.in_proj_weight = nn.Parameter(torch.empty(3 * hidden_dim, hidden_dim))
        self.in_proj_bias = nn.Parameter(torch.zeros(3 * hidden_dim))
        self.out_proj = bnn.Linear(hidden_dim, hidden_dim)
        nn.init.xavier_uniform_(self.in_proj_weight)
        nn.init.zeros_(self.out_proj.bias)

    def forward(self, x, B: int, S: int):
        qkv = bnn.linear(x, self, "in_proj_weight", "in_proj_bias")
        return self.out_proj(bnn.attention(qkv, B, S, self.num_heads, HEAD_DIM))


class _MLP(nn.Module):
    """torchvision's ``MLPBlock`` parameters (``0``: Linear with GELU, ``3``: Linear; 1, 2 and 4 hold none)."""

    def __init__(self, hidden_dim: int, mlp_dim: int):
        super().__init__()
        self.add_module("0", bnn.Linear(hidden_dim, mlp_dim, act="gelu_erf"))
        self.add_module("3", bnn.Linear(mlp_dim, hidden_dim))
        for m in (self[0], self[3]):
            nn.init.xavier_uniform_(m.weight)
            nn.init.normal_(m.bias, std=1e-6)

    def __getitem__(self, i: int) -> bnn.Linear:
        return self._modules[str(i)]

    def forward(self, x):
        return self[3](self[0](x))


class EncoderBlock(nn.Module):
    def __init__(self, num_heads: int, hidden_dim: int, mlp_dim: int, eps: float):
        super().__init__()
        self.ln_1 = bnn.LayerNorm(hidden_dim, eps)
        self.self_attention = _SelfAttention(hidden_dim, num_heads)
        self.ln_2 = bnn.LayerNorm(hidden_dim, eps)
        self.mlp = _MLP(hidden_dim, mlp_dim)


class Encoder(nn.Module):
    def __init__(self, seq_length: int, num_layers: int, num_heads: int, hidden_dim: int, mlp_dim: int, eps: float):
        super().__init__()
        self.pos_embedding = nn.Parameter(torch.empty(1, seq_length, hidden_dim).normal_(std=0.02))
        self.layers = nn.Sequential(OrderedDict(
            ("encoder_layer_{}".format(i), EncoderBlock(num_heads, hidden_dim, mlp_dim, eps)) for i in range(num_layers)))
        self.ln = bnn.LayerNorm(hidden_dim, eps)


class VisionTransformer(FederatedModule):
    """ViT classifier for ``[B, H, W, 3]`` NHWC images (bf16 on CUDA), fp32 logits.  ``hidden_dim / num_heads`` must be
    64 and the sequence ``(image_size / patch_size)^2 + 1`` at most 128 tokens (``ValueError`` otherwise), the shapes of
    the fused attention kernels."""
    loss_kind = "ce"
    head = "heads"
    default_lr = 0.01
    default_batch_size = 128
    is_vit = True          # parallel/features.py: the token kernel reads class_token / pos_embedding in fp32

    def __init__(self, image_size: int, patch_size: int, num_layers: int, num_heads: int, hidden_dim: int,
                 mlp_dim: int, num_classes: int = 10, name: Optional[str] = None):
        super().__init__()
        for k, v in (("image_size", image_size), ("patch_size", patch_size), ("num_layers", num_layers),
                     ("num_heads", num_heads), ("hidden_dim", hidden_dim), ("mlp_dim", mlp_dim),
                     ("num_classes", num_classes)):
            if isinstance(v, bool) or not isinstance(v, int) or v <= 0:
                raise ValueError("VisionTransformer: {} must be a positive int, got {!r}".format(k, v))
        if image_size % patch_size:
            raise ValueError("VisionTransformer: image_size {} is not divisible by patch_size {}".format(
                image_size, patch_size))
        seq = (image_size // patch_size) ** 2 + 1
        if seq > MAX_TOKENS:
            raise ValueError("VisionTransformer: {} tokens ({}^2 patches + the class token); the fused attention runs at "
                             "most {}".format(seq, image_size // patch_size, MAX_TOKENS))
        if hidden_dim != HEAD_DIM * num_heads:
            raise ValueError("VisionTransformer: hidden_dim / num_heads must be {}, got {} / {}".format(
                HEAD_DIM, hidden_dim, num_heads))
        self.name = name or "vit"
        self.image_size, self.patch_size, self.hidden_dim, self.seq_length = image_size, patch_size, hidden_dim, seq
        self.class_token = nn.Parameter(torch.zeros(1, 1, hidden_dim))
        self.conv_proj = _PatchEmbed(hidden_dim, patch_size)
        fan_in = 3 * patch_size * patch_size
        with torch.no_grad():
            nn.init.trunc_normal_(self.conv_proj.weight, std=math.sqrt(1.0 / fan_in))
        self.encoder = Encoder(seq, num_layers, num_heads, hidden_dim, mlp_dim, 1e-6)
        self.heads = nn.Sequential(OrderedDict(head=bnn.Linear(hidden_dim, num_classes, out_fp32=True)))
        nn.init.zeros_(self.heads.head.weight)
        nn.init.zeros_(self.heads.head.bias)

    def forward(self, x):
        """``x``: NHWC ``[B, H, W, 3]`` -> logits ``[B, num_classes]``."""
        if tuple(x.shape[1:]) != (self.image_size, self.image_size, 3):
            raise ValueError("VisionTransformer: expected [B, {0}, {0}, 3] images, got {1}".format(
                self.image_size, tuple(x.shape)))
        B, S, D = x.shape[0], self.seq_length, self.hidden_dim
        z = self.conv_proj(x).reshape(B, S - 1, D)
        s = bnn.vit_tokens(z, self.class_token, self.conv_proj.bias, self.encoder.pos_embedding).reshape(B * S, D)
        layers = list(self.encoder.layers)
        y = layers[0].ln_1(s)
        for i, blk in enumerate(layers):
            y, s = blk.ln_2.add_norm(blk.self_attention(y, B, S), s)
            nxt = layers[i + 1].ln_1 if i + 1 < len(layers) else self.encoder.ln
            y, s = nxt.add_norm(blk.mlp(y), s)
        return self.heads.head(y.view(B, S, D)[:, 0].contiguous())


def vit_tiny(num_classes: int = 10, image_size: int = 32, patch_size: int = 4) -> VisionTransformer:
    """ViT-Ti (DeiT-Tiny widths): D = 192, 12 layers, 3 heads, MLP 768."""
    return VisionTransformer(image_size, patch_size, 12, 3, 192, 768, num_classes, name="vit_tiny")


def vit_small(num_classes: int = 10, image_size: int = 32, patch_size: int = 4) -> VisionTransformer:
    """ViT-S: D = 384, 12 layers, 6 heads, MLP 1536."""
    return VisionTransformer(image_size, patch_size, 12, 6, 384, 1536, num_classes, name="vit_small")
