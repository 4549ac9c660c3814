"""Hand-written sm_90a kernels and the layers built on them.

``functional`` -- raw kernel wrappers (wgmma GEMM, fused SGD, im2col, ...)
``nn``         -- layers with hand-written backward passes (Linear, Conv2d,
                  BatchNorm2d(+residual+ReLU), LayerNorm, pooling, losses)
"""
from . import functional, nn
from ._ext import available, load
from .functional import (cast, fused_sgd, gather_rows, gemm, softmax_xent, weighted_sum_)

__all__ = ["functional", "nn", "available", "load", "gemm", "fused_sgd", "weighted_sum_", "cast",
           "gather_rows", "softmax_xent"]
