"""Layers built on the sm_90a kernels, with hand-written backward passes.

Every layer keeps an fp32 master parameter (a view into the flat parameter
arena once ``ParamArena`` has adopted the model) and consumes a bf16 shadow
copy (``weight_bf16``, a view into the bf16 arena refreshed by the fused SGD
kernel).  Backward kernels accumulate parameter gradients *directly* into
``param.grad`` (views of the flat gradient arena) and report ``None`` to
autograd, so there is no per-parameter accumulate kernel and the optimizer is a
single pass over the arena.

Layout: activations are bf16 NHWC / ``[rows, features]``.  Conv weights are
logically ``[Cout, Cin, KH, KW]`` (state_dict compatible with stock PyTorch)
stored channels_last, i.e. physically ``[Cout, KH, KW, Cin]`` -- exactly the
K-major B operand of the implicit GEMM.

On a CPU tensor every layer falls back to the equivalent ``torch.nn.functional``
call so the control plane / tests run on a GPU-less host.
"""
from __future__ import annotations

import contextlib
import math
from typing import Optional, Tuple

import torch
from torch import nn
from torch.nn import functional as TF

from . import functional as F
from ._ext import load

BF16 = torch.bfloat16


class _P:
    """Opaque holder that carries a Parameter through ``Function.apply`` WITHOUT making it a
    differentiable input.  In arena mode the backward kernels accumulate into ``param.grad`` themselves,
    so autograd must not see the leaf: its cached AccumulateGrad node remembers the stream it was
    created on, and merely scheduling it inside a CUDA-graph capture makes the engine record an event on
    that (uncaptured) stream -> cudaErrorStreamCaptureIsolation.  A fresh zero-size ``anchor`` leaf
    stands in so backward still runs for layers whose data input needs no gradient."""
    __slots__ = ("p",)

    def __init__(self, p):
        self.p = p


def _unwrap(v):
    return v.p if isinstance(v, _P) else v


def _wrap(param, x):
    """(holder-or-param, anchor-or-None) for one layer call."""
    return param if (param is None or _grad_target(param) is None) else _P(param)


def _anchor(x, *params):
    if any(p is not None and _grad_target(p) is not None for p in params) and torch.is_grad_enabled():
        return torch.empty(0, device=x.device, dtype=torch.float32, requires_grad=True)
    return None


class Ctx:
    """Stand-in for the autograd context: lets a hand-scheduled training step (``models/resnet.py``
    ``ResNet.explicit_step``) call the ``forward`` / ``backward`` bodies of the Functions below directly, in its own
    order and with its own fusions (two-piece gradients, parallel branches), without the autograd engine."""

    def __init__(self):
        self.saved_tensors = ()

    def save_for_backward(self, *tensors):
        self.saved_tensors = tensors

    def mark_non_differentiable(self, *a):
        pass


# dY[M, N] x X[M, K]: a weight-gradient GEMM above this many flops fills the machine on its own, gains nothing from a
# parallel branch and would only fight the persistent (one CTA per SM) dgrad kernels for SMs, so it runs inline
_WGRAD_OVERLAP_MAX_FLOPS = 4e9


class _WgradOverlap:
    """Weight-gradient GEMMs only feed the optimizer, so they are forked onto a side stream and overlap
    the dgrad -> BatchNorm-backward chain of the layers below (inside a captured graph this becomes a
    parallel branch).  Operand tensors are kept alive until the join so the caching allocator cannot hand
    their memory to the main stream early; the join is queued as an autograd end-of-backward callback and
    is also called by the trainer before the optimizer step."""

    def __init__(self):
        self.streams = {}
        self.keep = []
        self.pending = False
        self.queued = False

    def mark(self, ref):
        """Record "the operands are ready" on the current stream.  Calling this BEFORE the dgrad GEMM is enqueued and
        :meth:`run` (with the returned token) AFTER it puts the dgrad kernel -- the one on the critical path -- first
        in the captured graph's launch order while the weight-gradient branch still only depends on what precedes it."""
        if not ref.is_cuda:
            return None
        ev = torch.cuda.Event()
        ev.record(torch.cuda.current_stream(ref.device))
        return ev

    def run(self, fn, *keep, after=None):
        if not keep[0].is_cuda or 2.0 * keep[0].shape[0] * keep[0].shape[-1] * keep[1].shape[-1] > _WGRAD_OVERLAP_MAX_FLOPS:
            return fn()
        dev = keep[0].device
        side = self.streams.get(dev)
        if side is None:
            side = self.streams[dev] = torch.cuda.Stream(device=dev)
        cur = torch.cuda.current_stream(dev)
        if after is not None:
            side.wait_event(after)
        else:
            side.wait_stream(cur)
        with torch.cuda.stream(side):
            fn()
        self.keep.append(keep)
        self.pending = True
        if not self.queued:
            self.queued = True
            try:
                torch.autograd.Variable._execution_engine.queue_callback(self.join)
            except Exception:      # not inside a backward pass
                self.queued = False

    def join(self):
        self.queued = False
        if not self.pending:
            return
        for dev, side in self.streams.items():
            torch.cuda.current_stream(dev).wait_stream(side)
        self.keep.clear()
        self.pending = False


WGRAD = _WgradOverlap()


class _Branch:
    """Fork / join of an independent sub-chain (the shortcut conv + BN of a ResNet block, forward and backward) onto a
    side stream, so that inside a captured step it becomes a parallel graph branch.  These kernels use a fraction of
    the SMs and are latency bound, so two chains side by side cost the time of the longer one."""

    def __init__(self):
        self.streams = {}
        self.keep = []
        self.pending = False

    def fork(self, *keep):
        if not keep[0].is_cuda:
            return contextlib.nullcontext()
        dev = keep[0].device
        side = self.streams.get(dev)
        if side is None:
            side = self.streams[dev] = torch.cuda.Stream(device=dev)
        side.wait_stream(torch.cuda.current_stream(dev))
        self.keep.append(keep)
        self.pending = True
        return torch.cuda.stream(side)

    def join(self):
        if not self.pending:
            return
        for dev, side in self.streams.items():
            torch.cuda.current_stream(dev).wait_stream(side)
        self.keep.clear()
        self.pending = False


BRANCH = _Branch()


class _SgdEpilogue:
    """Optimizer epilogue of the convolution weight gradients.  While a trainer holds it open (:meth:`open`), a conv
    wgrad GEMM that owns complete gradient tiles (split-K = 1) applies the SGD step to the weights in its epilogue
    instead of accumulating into the gradient arena, and records what it updated: ``fused`` blocks
    ``(offset, rows, cols, ld)`` and, for centre-tap convolutions, the ``nograd`` range ``(offset, length)`` of the whole
    weight (its other taps never receive a gradient).  The trainer's leftover optimizer pass covers the rest of the
    arena (``F.sgd_segments``).  The gradient of a fused block is never written, so it stays zero for unfused steps.
    ``prox``: FedProx step anchored on ``arena.global_w`` (``hyper`` then holds the coefficient as its fifth float).
    ``corr``: SCAFFOLD step with the correction ``c - c_i`` (fp32, indexed like the parameters).
    ``adam_v``: AdamW step with this second moment (``arena.momentum`` is the first, ``hyper`` the step's AdamW row).
    ``fuse=False`` (a gradient-clipped step, whose coefficient needs the whole gradient): no GEMM applies the step;
    only the ``nograd`` ranges are recorded -- the centre-tap weights minus their centre tap."""

    def __init__(self):
        self.arena = None
        self.fuse = True

    @contextlib.contextmanager
    def open(self, arena, hyper, nesterov, prox=False, corr=None, adam_v=None, fuse=True):
        self.arena, self.hyper, self.nesterov, self.fuse = arena, hyper, nesterov, fuse
        self.anchor = arena.global_w if prox else None
        self.corr = corr
        self.adam_v = adam_v
        self.fused, self.nograd = [], []
        try:
            yield self
        finally:
            self.arena = None

    @property
    def active(self):
        """True while wgrad GEMMs apply the optimizer step in their epilogue."""
        return self.arena is not None and self.fuse

    @property
    def recording(self):
        """True while an unfused step records its no-gradient ranges."""
        return self.arena is not None and not self.fuse

    def args(self, out2d):
        """``sgd=`` argument for a wgrad GEMM writing the arena gradient view ``out2d``, or None when not fusing."""
        a = self.arena
        if not self.active:
            return None
        return F.sgd_epilogue_args(a.theta, a.grad, out2d, self.hyper, a.momentum, a.theta_bf16, self.nesterov,
                                   self.anchor, self.corr, self.adam_v)

    def record(self, out2d, nograd_of=None):
        off = (out2d.data_ptr() - self.arena.grad.data_ptr()) // 4
        self.fused.append((off, out2d.shape[0], out2d.shape[1], out2d.stride(0)))
        if nograd_of is not None:
            self.nograd.append(((nograd_of.data_ptr() - self.arena.grad.data_ptr()) // 4, nograd_of.numel()))

    def record_nograd(self, out2d, nograd_of):
        """Unfused step: the ranges of the weight gradient ``nograd_of`` outside the block ``out2d`` (the centre tap,
        which the GEMM accumulated into the arena) as ``nograd`` ranges."""
        g0 = self.arena.grad.data_ptr()
        pos = (nograd_of.data_ptr() - g0) // 4
        end = pos + nograd_of.numel()
        off, ld, cols = (out2d.data_ptr() - g0) // 4, out2d.stride(0), out2d.shape[1]
        for r in range(out2d.shape[0]):
            s = off + r * ld
            if s > pos:
                self.nograd.append((pos, s - pos))
            pos = s + cols
        if pos < end:
            self.nograd.append((pos, end - pos))


SGD_EPI = _SgdEpilogue()


def _wgrad(fn, out2d, nograd_of=None):
    """Run a weight-gradient GEMM ``fn(sgd)`` -- with the optimizer epilogue when it is open and the GEMM accepts it,
    accumulating into ``out2d`` otherwise."""
    sgd = SGD_EPI.args(out2d)
    if sgd is not None and fn(sgd):
        SGD_EPI.record(out2d, nograd_of)
    else:
        fn(None)
        if nograd_of is not None and SGD_EPI.recording:
            SGD_EPI.record_nograd(out2d, nograd_of)


def _grad_target(p: Optional[torch.Tensor]):
    """fp32 gradient buffer to accumulate into (arena view) or None."""
    if p is None or p.grad is None or p.grad.dtype != torch.float32:
        return None
    return p.grad


def _shadow(module: nn.Module, name: str, param: torch.Tensor, as2d: bool = True) -> torch.Tensor:
    """bf16 copy of a parameter.  Arena-adopted modules carry ``<name>_bf16``
    views that the SGD / FedAvg kernels keep in sync; otherwise cast on the fly."""
    sh = getattr(module, name + "_bf16", None)
    if sh is not None:
        return sh
    if param.dim() == 4:  # channels_last conv weight -> [Cout, KH*KW*Cin]
        src = param.detach().permute(0, 2, 3, 1).contiguous()
        return F.cast(src.view(param.shape[0], -1), BF16)
    return F.cast(param.detach().contiguous(), BF16)


# ================================================================================ Linear
class _LinearFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, weight, bias, w_bf16, act, out_fp32, flags_cfg, anchor):
        weight, bias = _unwrap(weight), _unwrap(bias)
        x2 = x.reshape(-1, x.shape[-1])
        kw = {}
        if flags_cfg is not None:
            kw = dict(flags=flags_cfg["flags"], flag_epoch=flags_cfg.get("epoch", 0), flag_elem_off=flags_cfg["elem_off"],
                      flag_tile_elems=flags_cfg["tile_elems"], flag_bias_off=flags_cfg.get("bias_off", -1),
                      force_bn=128, flag_epoch_word=flags_cfg.get("epoch_word"))
        y = F.gemm(x2, w_bf16, bias=bias, act=act if act == 1 else 0,
                   out_dtype=torch.float32 if out_fp32 else BF16, **kw)
        ctx.act = act
        pre = None
        if act in (2, 3):  # GELU needs the pre-activation for backward
            pre = y
            y = F.gelu(pre) if act == 2 else F.gelu_erf(pre)
        ctx.save_for_backward(x2, w_bf16, y if act == 1 else pre)
        ctx.weight, ctx.bias = weight, bias
        ctx.x_shape = x.shape
        ctx.needs_dx = x.requires_grad
        return y.view(*x.shape[:-1], w_bf16.shape[0])

    @staticmethod
    def backward(ctx, dy):
        x2, w_bf16, aux = ctx.saved_tensors
        dy2 = dy.reshape(-1, dy.shape[-1])
        if dy2.dtype != BF16:
            dy2 = F.cast(dy2.contiguous(), BF16)
        elif not dy2.is_contiguous():
            dy2 = dy2.contiguous()
        if ctx.act == 1:
            dy2 = F.relu_bwd(aux, dy2)
        elif ctx.act == 2:
            dy2 = F.gelu_bwd(aux, dy2)
        elif ctx.act == 3:
            dy2 = F.gelu_erf_bwd(aux, dy2)
        gw, gb = _linear_param_grads(dy2, x2, ctx.weight, ctx.bias)
        dx = None
        if ctx.needs_dx:
            # dgrad: dX[M, K] = dY[M, N] W[N, K]   (B = W is MN-major for this product)
            dx = F.gemm(dy2, w_bf16, b_mn=True).view(ctx.x_shape)
        return dx, gw, gb, None, None, None, None, None


def _act_bwd(ctx, dy, aux):
    """``dY'``: the bf16 gradient of a Linear's pre-activation output."""
    dy2 = dy.reshape(-1, dy.shape[-1])
    if dy2.dtype != BF16:
        dy2 = F.cast(dy2.contiguous(), BF16)
    elif not dy2.is_contiguous():
        dy2 = dy2.contiguous()
    if ctx.act == 1:
        dy2 = F.relu_bwd(aux, dy2)
    elif ctx.act == 2:
        dy2 = F.gelu_bwd(aux, dy2)
    return dy2


def _frozen(p) -> bool:
    return p is None or not p.requires_grad


def _linear_param_grads(dy2, x2, weight, bias):
    """Weight and bias gradients of a Linear: accumulated into the arena views (returns None, None) or returned to
    autograd.  A frozen weight runs no weight-gradient GEMM, a frozen bias no column sum."""
    gw = gb = None
    if not _frozen(weight):
        # wgrad: dW[N, K] += dY^T[N, M] X[M, K]   (both operands MN-major, no transposes)
        tgt = _grad_target(weight)
        if tgt is not None:
            out2d = tgt.view(weight.shape[0], -1)
            WGRAD.run(lambda: F.gemm(dy2, x2, a_mn=True, b_mn=True, out=out2d, accumulate=True), dy2, x2)
        else:
            gw = F.gemm(dy2, x2, a_mn=True, b_mn=True, out_dtype=torch.float32, accumulate=True).view_as(weight)
    if not _frozen(bias):
        tb = _grad_target(bias)
        if tb is not None:
            F.colsum_(dy2, tb, accumulate=True)
        else:
            gb = F.colsum_(dy2, torch.zeros_like(bias, dtype=torch.float32), accumulate=True)
    return gw, gb


def _grad_or_scratch(p):
    """(buffer to accumulate into, gradient to return to autograd) of a trainable parameter."""
    tgt = _grad_target(p)
    if tgt is not None:
        return tgt, None
    g = torch.zeros_like(p, dtype=torch.float32)
    return g, g


class _LoraLinearFn(torch.autograd.Function):
    """``y = act(x W^T + b + s (x A^T) B^T)`` with the rank term per targeted output slice (``Linear.add_lora``):
    the down projection ``U = x A^T`` is one launch for every slice, the up projection runs in the epilogue of the
    base GEMM, and the output is rounded once.  Backward: ``V = dY' B`` (one launch), ``dx = dY' W + s V A`` (the
    same epilogue form), ``dB = s dY'^T U`` and ``dA = s V^T x`` as fixed-order reductions over the rows."""

    @staticmethod
    def forward(ctx, x, weight, bias, w_bf16, lora_a, lora_b, a_bf16, b_bf16, cfg, act, out_fp32, anchor):
        weight, bias, lora_a, lora_b = _unwrap(weight), _unwrap(bias), _unwrap(lora_a), _unwrap(lora_b)
        x2 = x.reshape(-1, x.shape[-1])
        r, s, slot, ds = cfg
        R, K = a_bf16.shape
        u = F.lora_down(x2, a_bf16, T=1, rs=R, kt=K, xoff=(0,), w_ts=0, wsj=K, wsk=1)
        y = F.gemm_lora(x2, w_bf16, dict(u=u, f=b_bf16, fs_n=r, fs_j=1, rs=r, ds=ds, slot=slot, s=s), bias=bias,
                        act=act if act != 2 else 0, out_dtype=torch.float32 if out_fp32 else BF16)
        pre = None
        if act == 2:
            pre = y
            y = F.gelu(pre)
        ctx.save_for_backward(x2, w_bf16, u, a_bf16, b_bf16, y if act == 1 else pre)
        ctx.act, ctx.cfg = act, cfg
        ctx.weight, ctx.bias, ctx.lora_a, ctx.lora_b = weight, bias, lora_a, lora_b
        ctx.x_shape = x.shape
        ctx.needs_dx = x.requires_grad
        return y.view(*x.shape[:-1], w_bf16.shape[0])

    @staticmethod
    def backward(ctx, dy):
        x2, w_bf16, u, a_bf16, b_bf16, aux = ctx.saved_tensors
        dy2 = _act_bwd(ctx, dy, aux)
        r, s, slot, ds = ctx.cfg
        R, K = a_bf16.shape
        gw, gb = _linear_param_grads(dy2, x2, ctx.weight, ctx.bias)
        sl = [i for i in range(3) if slot[i] >= 0]          # targeted slices in rank-block order
        sl.sort(key=lambda i: slot[i])
        lo = [i * ds for i in sl]
        v = F.lora_down(dy2, b_bf16, T=len(sl), rs=r, kt=ds, xoff=lo, w_ts=ds * r, wsj=1, wsk=r)
        ga = gbb = None
        if not _frozen(ctx.lora_b):
            tgt, gbb = _grad_or_scratch(ctx.lora_b)
            F.lora_grad_(dy2, u, tgt, NA=ds, NB=r, lo=lo, qo=[slot[i] * r for i in sl], osa=r, osb=1, out_ts=ds * r,
                         s=s)
        if not _frozen(ctx.lora_a):
            tgt, ga = _grad_or_scratch(ctx.lora_a)
            F.lora_grad_(x2, v, tgt, NA=K, NB=R, lo=(0,), qo=(0,), osa=1, osb=K, out_ts=0, s=s)
        dx = None
        if ctx.needs_dx:
            dx = F.gemm_lora(dy2, w_bf16, dict(u=v, f=a_bf16, fs_n=1, fs_j=K, rs=R, ds=K, slot=(0, -1, -1), s=s),
                             b_mn=True).view(ctx.x_shape)
        return dx, gw, gb, None, ga, gbb, None, None, None, None, None, None


class Linear(nn.Module):
    """``y = act(x W^T + b)``; ``act`` in {None, 'relu', 'gelu', 'gelu_erf'}: ReLU is fused into the GEMM epilogue,
    the tanh GELU ('gelu') and the exact one ('gelu_erf', ``torch.nn.GELU()``) run as an elementwise kernel after it."""

    def __init__(self, in_features: int, out_features: int, bias: bool = True, act: Optional[str] = None,
                 out_fp32: bool = False):
        super().__init__()
        self.in_features, self.out_features = in_features, out_features
        self.act = {None: 0, "relu": 1, "gelu": 2, "gelu_erf": 3}[act]
        self.out_fp32 = out_fp32
        self.weight = nn.Parameter(torch.empty(out_features, in_features))
        self.bias = nn.Parameter(torch.empty(out_features)) if bias else None
        self.flags_cfg = None  # set by FedAvgSession for the first layer (bcast_gemm)
        self.reset_parameters()

    def reset_parameters(self):
        nn.init.kaiming_uniform_(self.weight, a=math.sqrt(5))
        if self.bias is not None:
            bound = 1 / math.sqrt(self.in_features)
            nn.init.uniform_(self.bias, -bound, bound)

    def add_lora(self, r: int, s: float, targets: Tuple[bool, ...]) -> None:
        """Low-rank adapters on the output slices ``targets`` (the output splits into ``len(targets)`` equal slices, at
        most three: the packed q / k / v projection): ``lora_A`` ``[T r, in]`` stacks the targeted slices' ``A`` in slice
        order, ``lora_B`` ``[T ds, r]`` their ``B``.  ``A`` starts as ``kaiming_uniform_(a=sqrt(5))``, ``B`` at zero, so
        the layer computes what it did.  Called before the arena adopts the model."""
        n = len(targets)
        if not 1 <= n <= 3 or self.out_features % n or not any(targets):
            raise ValueError("LoRA: one to three equal output slices with at least one target, got {}".format(targets))
        ds = self.out_features // n
        if ds % 32 or self.in_features % 32:
            raise ValueError("LoRA needs slice widths and in_features that are multiples of 32")
        slot, t = [-1, -1, -1], 0
        for i, on in enumerate(targets):
            if on:
                slot[i], t = t, t + 1
        a = torch.empty(t * r, self.in_features)
        for i in range(t):
            nn.init.kaiming_uniform_(a[i * r:(i + 1) * r], a=math.sqrt(5))
        self.lora_A = nn.Parameter(a)
        self.lora_B = nn.Parameter(torch.zeros(t * ds, r))
        self.lora_cfg = (int(r), float(s), tuple(slot), ds)

    def _lora_term(self, x):
        """CPU form of the adapter term, ``s (x A_t^T) B_t^T`` in the targeted slices and zero elsewhere."""
        r, s, slot, ds = self.lora_cfg
        u = x @ self.lora_A.to(x.dtype).t()
        parts = []
        for t in slot:
            if t < 0:
                parts.append(x.new_zeros(*x.shape[:-1], ds))
            else:
                parts.append(s * (u[..., t * r:(t + 1) * r] @ self.lora_B[t * ds:(t + 1) * ds].to(x.dtype).t()))
        return torch.cat(parts[: self.out_features // ds], dim=-1)

    def forward(self, x):
        lora = getattr(self, "lora_cfg", None)
        if not x.is_cuda:
            y = TF.linear(x, self.weight.to(x.dtype), None if self.bias is None else self.bias.to(x.dtype))
            if lora is not None:
                y = y + self._lora_term(x)
            if self.act == 3:
                return TF.gelu(y, approximate="none")
            return TF.relu(y) if self.act == 1 else (TF.gelu(y, approximate="tanh") if self.act == 2 else y)
        if x.dtype != BF16:
            x = F.cast(x.contiguous(), BF16)
        if lora is not None:
            if self.act == 3:
                raise ValueError("LoRA adapters on a Linear with act='gelu_erf' are not supported")
            y = _LoraLinearFn.apply(x, _wrap(self.weight, x), _wrap(self.bias, x), _shadow(self, "weight", self.weight),
                                    _wrap(self.lora_A, x), _wrap(self.lora_B, x), _shadow(self, "lora_A", self.lora_A),
                                    _shadow(self, "lora_B", self.lora_B), lora, self.act, self.out_fp32,
                                    _anchor(x, self.lora_A, self.lora_B))
            return y
        if getattr(self, "fp8", False) and self.act == 0 and self.bias is None and not self.out_fp32:
            y = matmul_fp8(x.reshape(-1, x.shape[-1]), self, _shadow(self, "weight", self.weight), self.in_features)
            return y.view(*x.shape[:-1], self.out_features)
        cfg = self.flags_cfg
        if cfg is not None and cfg.get("epoch_word") is None:
            self.flags_cfg = None  # launch-constant epoch: one-shot, only the first GEMM after a round is gated
        return _LinearFn.apply(x, _wrap(self.weight, x), _wrap(self.bias, x), _shadow(self, "weight", self.weight),
                               self.act, self.out_fp32, cfg, _anchor(x, self.weight, self.bias))


def linear(x: torch.Tensor, owner: nn.Module, weight: str, bias: str) -> torch.Tensor:
    """``x W^T + b`` with ``W = owner.<weight>`` and ``b = owner.<bias>``: the GEMM of :class:`Linear` for a module
    that keeps its projection under other ``state_dict`` names (torchvision's packed ``in_proj_weight`` /
    ``in_proj_bias``).  The arena's bf16 shadow is ``owner.<weight>_bf16``."""
    w, b = getattr(owner, weight), getattr(owner, bias)
    if not x.is_cuda:
        return TF.linear(x, w.to(x.dtype), b.to(x.dtype))
    if x.dtype != BF16:
        x = F.cast(x.contiguous(), BF16)
    return _LinearFn.apply(x, _wrap(w, x), _wrap(b, x), _shadow(owner, weight, w), 0, False, None, _anchor(x, w, b))


# ================================================================================ Conv2d (NHWC, implicit GEMM)
class _ConvFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, weight, w_bf16, plan, anchor, stats=None, gate=None):
        """``plan``: GEMM lowering of this call (``F.conv_plan``).  ``gate``: bcast_gemm arrival-flag configuration of
        this layer's weights (first conv of the model only)."""
        y, col = F.conv_fwd(x, w_bf16, plan, col_stats=stats, gate=gate)
        ctx.igemm = plan.form == "implicit" and y is not None      # col IS x: the wgrad gathers im2col(x) on the fly
        if plan.form == "implicit" and y is None:                  # the kernel declined this shape: explicit im2col
            y, col = F.conv_fwd(x, w_bf16, plan, form="im2col", col_stats=stats, gate=gate)
        ctx.save_for_backward(col, w_bf16)
        ctx.weight, ctx.plan = _unwrap(weight), plan
        ctx.needs_dx = x.requires_grad
        return y.view(plan.n, plan.ho, plan.wo, plan.cout)

    @staticmethod
    def backward(ctx, dy):
        col, w_bf16 = ctx.saved_tensors
        p = ctx.plan
        dy2 = dy.reshape(p.M, p.cout)
        if not dy2.is_contiguous():
            dy2 = dy2.contiguous()
        k_true = p.kh * p.kw * p.c
        g2 = None
        tgt = _grad_target(ctx.weight)
        if p.form == "centre" and tgt is None:
            # only the centre tap receives a gradient; the other taps of the full weight gradient stay zero
            g2 = torch.zeros((p.cout, k_true), dtype=torch.float32, device=dy.device)
            F.gemm(dy2, col, a_mn=True, b_mn=True, out=p.weight(g2), accumulate=True)
        tok = WGRAD.mark(dy2)      # the weight-gradient branch depends on what is enqueued so far, not on the dgrad below
        dx = None
        if ctx.needs_dx:
            if p.dgrad == "implicit":
                dx = F.conv_igemm_dgrad(dy2.view(p.n, p.ho, p.wo, p.cout), w_bf16, (p.n, p.h, p.w, p.c), p.kh, p.kw,
                                        p.pad, stride=p.stride)
            if dx is None:
                dcol = F.gemm(dy2, p.weight(w_bf16), b_mn=True)  # [M, K]
                dx = dcol.view(p.n, p.h, p.w, p.c) if p.dgrad == "view" else \
                    F.col2im(dcol, (p.n, p.h, p.w, p.c), p.kh, p.kw, p.stride, p.pad, p.ho, p.wo)
        if tgt is not None:
            # the arena view is channels_last: physical [Cout, KH, KW, Cin] == [Cout, K]
            out2d = tgt.permute(0, 2, 3, 1).reshape(p.cout, k_true) if tgt.dim() == 4 else tgt.view(p.cout, k_true)
            assert out2d.data_ptr() == tgt.data_ptr(), "conv weight grad must be channels_last in the arena"
            # an optimizer epilogue rewrites the bf16 weights the dgrad above reads: it must start after it
            if p.form == "centre":
                g2d = p.weight(out2d)
                WGRAD.run(lambda: _wgrad(lambda sgd: F.gemm(dy2, col, a_mn=True, b_mn=True, out=g2d, accumulate=True,
                                                            sgd=sgd) is not None, g2d, nograd_of=tgt),
                          dy2, col, after=None if SGD_EPI.active else tok)
            elif ctx.igemm:
                WGRAD.run(lambda: _wgrad(lambda sgd: F.conv_igemm_wgrad_(dy2, col, out2d, p.kh, p.kw, p.stride, p.pad,
                                                                         sgd=sgd), out2d),
                          dy2, col, after=None if SGD_EPI.active else tok)
            else:
                WGRAD.run(lambda: F.gemm(dy2, col, a_mn=True, b_mn=True, out=out2d, accumulate=True, n_valid=k_true),
                          dy2, col, after=tok)
        elif ctx.igemm:
            g2 = torch.zeros((p.cout, k_true), dtype=torch.float32, device=dy.device)
            F.conv_igemm_wgrad_(dy2, col, g2, p.kh, p.kw, p.stride, p.pad)
        elif p.form != "centre":
            g2 = F.gemm(dy2, col, a_mn=True, b_mn=True, out_dtype=torch.float32, accumulate=True, n_valid=k_true)
        gw = None if g2 is None else g2.view(p.cout, p.kh, p.kw, p.c).permute(0, 3, 1, 2)
        return dx, gw, None, None, None, None, None


class Conv2d(nn.Module):
    """NHWC convolution (no bias -- every conv in ResNet is followed by BatchNorm)."""

    def __init__(self, in_channels: int, out_channels: int, kernel_size: int, stride: int = 1, padding: int = 0):
        super().__init__()
        self.in_channels, self.out_channels = in_channels, out_channels
        self.kernel_size, self.stride, self.padding = kernel_size, stride, padding
        w = torch.empty(out_channels, in_channels, kernel_size, kernel_size)
        nn.init.kaiming_normal_(w, mode="fan_out", nonlinearity="relu")
        self.weight = nn.Parameter(w.contiguous(memory_format=torch.channels_last))
        self.k_true = kernel_size * kernel_size * in_channels
        self.kp = F.im2col_k(kernel_size, kernel_size, in_channels)
        self.flags_cfg = None   # bcast_gemm: set by FedAvgSession.gate_first_conv for the first conv of the model

    def _w_bf16(self, gated: bool = True):
        """bf16 ``[Cout, kp]`` weights.  ``gated=False``: the zero-padded copy does not wait on the first layer's
        arrival flags (callers that run after the round-end collective has been joined)."""
        sh = getattr(self, "weight_bf16", None)
        if sh is None:
            sh = _shadow(self, "weight", self.weight)
        sh = sh.view(self.out_channels, self.k_true)
        if self.kp != self.k_true:  # K not a multiple of 8 (7x7x3 stem): zero-padded copy for TMA
            sh = F.pad_rows(sh, self.kp, gate=self.flags_cfg if gated else None)
        return sh

    def forward(self, x):
        if not x.is_cuda:
            y = TF.conv2d(x.permute(0, 3, 1, 2), self.weight.to(x.dtype), None, self.stride, self.padding)
            return y.permute(0, 2, 3, 1)
        if getattr(self, "fp8", False):
            return conv2d_fp8(x, self)
        stats = self._fusable_stats(x)
        y = _ConvFn.apply(x, _wrap(self.weight, x), self._w_bf16(), self.plan(x), _anchor(x, self.weight), stats,
                          self.flags_cfg)
        if stats is not None:
            y._bn_stats_ws = stats      # tells the BatchNorm that owns this workspace to skip its statistics pass
        return y

    def plan(self, x) -> F.ConvPlan:
        n, h, w, c = x.shape
        return F.conv_plan(n, h, w, c, self.out_channels, self.kernel_size, self.kernel_size, self.stride,
                           self.padding)

    def _fusable_stats(self, x):
        """The following BatchNorm's statistics workspace (``bn_ws``, linked by the model) if this call's GEMM
        can accumulate the batch statistics in its epilogue; ``None`` otherwise."""
        ws = getattr(self, "bn_ws", None)
        if ws is None or not self.training or not torch.is_grad_enabled():
            return None
        p = self.plan(x)
        return ws[: 2 * p.cout] if F.gemm_stats_fusable(p.M, p.cout, p.K) else None


# ================================================================================ BatchNorm (+residual +ReLU)
class _BNFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, residual, gamma, beta, rmean, rvar, nbt, eps, momentum, relu, training, ws, anchor,
                stats_ready=False):
        gamma, beta = _unwrap(gamma), _unwrap(beta)
        C_ = load()
        c = x.shape[-1]
        rows = x.numel() // c
        y = torch.empty_like(x)
        if ws is None:
            ws = torch.zeros(4 * c, dtype=torch.float32, device=x.device)
        sums_f, sums_b = ws[: 2 * c], ws[2 * c:]
        save_mean = torch.empty(c, dtype=torch.float32, device=x.device)
        save_rstd = torch.empty(c, dtype=torch.float32, device=x.device)
        if training and not stats_ready:     # stats_ready: the producing GEMM's epilogue already accumulated them
            C_.bn_stats(x, sums_f, rows, c)
        C_.bn_apply(x, residual, y, sums_f, gamma, beta, rmean, rvar, save_mean, save_rstd, nbt, rows, c, eps,
                    momentum, relu, training)
        ctx.save_for_backward(x, y, save_mean, save_rstd)
        ctx.gamma, ctx.beta, ctx.sums_b = gamma, beta, sums_b
        ctx.relu, ctx.has_res, ctx.rows, ctx.c = relu, residual is not None, rows, c
        return y

    @staticmethod
    def backward(ctx, dy, dy_b=None):
        """``dy_b``: optional second piece of the incoming gradient (``dy + dy_b``), summed inside the kernel --
        only the hand-scheduled step passes it (autograd sums gradients itself)."""
        C_ = load()
        x, y, mean, rstd = ctx.saved_tensors
        if not dy.is_contiguous():
            dy = dy.contiguous()
        gamma, beta = ctx.gamma, ctx.beta
        dx = torch.empty_like(x)
        dres = torch.empty_like(x) if ctx.has_res else None
        tg, tb = _grad_target(gamma), _grad_target(beta)
        gg = gb = None
        if tg is None:
            gg = tg = torch.zeros(ctx.c, dtype=torch.float32, device=x.device)
        if tb is None:
            gb = tb = torch.zeros(ctx.c, dtype=torch.float32, device=x.device)
        # one launch (a thread-block cluster per 16-channel slice, csrc/norm.cu); shapes it declines take reduce + apply
        if not C_.bn_bwd_cluster(x, y, dy, dy_b, dx, dres, gamma, mean, rstd, tg, tb, ctx.rows, ctx.c, ctx.relu, 16):
            if dy_b is not None:
                dy = F.add(dy, dy_b.contiguous())
            C_.bn_bwd_reduce(x, y, dy, mean, rstd, ctx.sums_b, ctx.rows, ctx.c, ctx.relu)
            C_.bn_bwd_apply(x, y, dy, dx, dres, gamma, mean, rstd, ctx.sums_b, tg, tb, ctx.rows, ctx.c, ctx.relu)
        if ctx.has_res and dres is None:
            dres = dy
        return dx, dres, gg, gb, None, None, None, None, None, None, None, None, None, None


class BatchNorm2d(nn.Module):
    """BatchNorm over the channel (last) axis of an NHWC tensor with the residual add
    and ReLU of a ResNet block fused into the same pass:  ``relu(bn(x) + residual)``."""

    def __init__(self, num_features: int, eps: float = 1e-5, momentum: float = 0.1, relu: bool = False):
        super().__init__()
        self.num_features, self.eps, self.momentum, self.relu = num_features, eps, momentum, relu
        self.weight = nn.Parameter(torch.ones(num_features))
        self.bias = nn.Parameter(torch.zeros(num_features))
        self.register_buffer("running_mean", torch.zeros(num_features))
        self.register_buffer("running_var", torch.ones(num_features))
        self.register_buffer("num_batches_tracked", torch.tensor(0, dtype=torch.long))
        self.workspace = None  # [4*C] fp32 slice of the model-wide stats workspace (zeroed once per step)

    def forward(self, x, residual=None):
        if not x.is_cuda:
            xn = x.permute(0, 3, 1, 2)
            y = TF.batch_norm(xn, self.running_mean, self.running_var, self.weight, self.bias, self.training,
                              self.momentum, self.eps).permute(0, 2, 3, 1)
            if self.training:
                self.num_batches_tracked += 1
            if residual is not None:
                y = y + residual
            return TF.relu(y) if self.relu else y
        ws = self.workspace
        if ws is None:
            ws = torch.zeros(4 * self.num_features, dtype=torch.float32, device=x.device)
        fused = getattr(x, "_bn_stats_ws", None)      # set by the producing Conv2d when its GEMM took the statistics
        ready = (fused is not None and self.workspace is not None and self.training
                 and fused.data_ptr() == self.workspace.data_ptr())
        return _BNFn.apply(x, residual, _wrap(self.weight, x), _wrap(self.bias, x), self.running_mean,
                           self.running_var, self.num_batches_tracked if self.training else None, self.eps,
                           self.momentum, self.relu, self.training, ws, _anchor(x, self.weight), ready)


# ================================================================================ GroupNorm (+residual +ReLU)
class _GNFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, residual, gamma, beta, groups, eps, relu, need_bwd, anchor):
        """``need_bwd``: allocate the backward's scratch (``F.gn_work``), whose counters the forward kernel zeroes."""
        gamma, beta = _unwrap(gamma), _unwrap(beta)
        work = F.gn_work(x.shape[0], x.shape[3], groups, x.device) if need_bwd else None
        y, mean, rstd = F.gn_fwd(x, residual, gamma, beta, groups, eps, relu, work)
        ctx.save_for_backward(x, y, mean, rstd, work)
        ctx.gamma, ctx.beta = gamma, beta
        ctx.groups, ctx.relu, ctx.has_res = groups, relu, residual is not None
        return y

    @staticmethod
    def backward(ctx, dy, dy_b=None):
        """``dy_b``: optional second piece of the incoming gradient, summed inside the kernel (hand-scheduled step only)."""
        x, y, mean, rstd, work = ctx.saved_tensors
        gamma, beta = ctx.gamma, ctx.beta
        tg, tb = _grad_target(gamma), _grad_target(beta)
        gg = gb = None
        if tg is None:
            gg = tg = torch.zeros(x.shape[3], dtype=torch.float32, device=x.device)
        if tb is None:
            gb = tb = torch.zeros(x.shape[3], dtype=torch.float32, device=x.device)
        dx, dres = F.gn_bwd(x, y, dy, dy_b, gamma, mean, rstd, tg, tb, ctx.groups, ctx.relu, want_dres=ctx.has_res,
                            work=work)
        return dx, dres, gg, gb, None, None, None, None, None


class GroupNorm(nn.Module):
    """GroupNorm over ``num_groups`` contiguous channel blocks of an NHWC tensor (``torch.nn.GroupNorm``'s grouping and
    ``weight`` / ``bias``, no buffers), with the residual add and ReLU of a ResNet block fused into the same pass:
    ``relu(gn(x) + residual)``.  Statistics are per sample, so training and evaluation compute the same thing."""

    def __init__(self, num_groups: int, num_channels: int, eps: float = 1e-5, relu: bool = False):
        super().__init__()
        if (isinstance(num_groups, bool) or not isinstance(num_groups, int) or num_groups <= 0
                or num_channels % num_groups):
            raise ValueError("GroupNorm: num_groups must be a positive int dividing num_channels, got {!r} for {} "
                             "channels".format(num_groups, num_channels))
        self.num_groups, self.num_channels, self.eps, self.relu = num_groups, num_channels, eps, relu
        self.weight = nn.Parameter(torch.ones(num_channels))
        self.bias = nn.Parameter(torch.zeros(num_channels))

    def forward(self, x, residual=None):
        if not x.is_cuda:
            y = TF.group_norm(x.permute(0, 3, 1, 2), self.num_groups, self.weight, self.bias,
                              self.eps).permute(0, 2, 3, 1)
            if residual is not None:
                y = y + residual
            return TF.relu(y) if self.relu else y
        return _GNFn.apply(x.contiguous(), residual, _wrap(self.weight, x), _wrap(self.bias, x), self.num_groups,
                           self.eps, self.relu, torch.is_grad_enabled(), _anchor(x, self.weight))


# ================================================================================ pooling / misc
class _MaxPoolFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, k, stride, pad):
        y, arg = F.maxpool(x, k, stride, pad)
        ctx.save_for_backward(arg)
        ctx.cfg = (tuple(x.shape), k, stride, pad)
        return y

    @staticmethod
    def backward(ctx, dy, dy_b=None):
        (arg,) = ctx.saved_tensors
        shape, k, stride, pad = ctx.cfg
        return F.maxpool_bwd(dy.contiguous(), arg, shape, k, stride, pad, dy_b=dy_b), None, None, None


class MaxPool2d(nn.Module):
    def __init__(self, kernel_size: int = 3, stride: int = 2, padding: int = 1):
        super().__init__()
        self.k, self.stride, self.pad = kernel_size, stride, padding

    def forward(self, x):
        if not x.is_cuda:
            return TF.max_pool2d(x.permute(0, 3, 1, 2), self.k, self.stride, self.pad).permute(0, 2, 3, 1)
        return _MaxPoolFn.apply(x, self.k, self.stride, self.pad)


class _AvgPoolFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x):
        ctx.shape = tuple(x.shape)
        return F.avgpool(x)

    @staticmethod
    def backward(ctx, dy):
        return F.avgpool_bwd(dy.contiguous(), ctx.shape)


class GlobalAvgPool(nn.Module):
    """NHWC ``[N,H,W,C] -> [N,C]`` (a view when H = W = 1, the 32x32-input ResNet case)."""

    def forward(self, x):
        if x.shape[1] == 1 and x.shape[2] == 1:
            return x.reshape(x.shape[0], x.shape[3])
        if not x.is_cuda:
            return x.mean(dim=(1, 2))
        return _AvgPoolFn.apply(x)


# ================================================================================ LayerNorm / GELU / softmax
class _LNFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, residual, gamma, beta, eps, anchor):
        gamma, beta = _unwrap(gamma), _unwrap(beta)
        C_ = load()
        c = x.shape[-1]
        rows = x.numel() // c
        y = torch.empty_like(x)
        mean = torch.empty(rows, dtype=torch.float32, device=x.device)
        rstd = torch.empty(rows, dtype=torch.float32, device=x.device)
        C_.layernorm_fwd(x, residual, y, gamma, beta, mean, rstd, rows, c, eps)
        pre = x if residual is None else F.add(x, residual)
        ctx.save_for_backward(pre, mean, rstd)
        ctx.gamma, ctx.beta, ctx.has_res, ctx.rows, ctx.c = gamma, beta, residual is not None, rows, c
        return y

    @staticmethod
    def backward(ctx, dy):
        C_ = load()
        pre, mean, rstd = ctx.saved_tensors
        dy = dy.contiguous()
        dx = torch.empty_like(pre)
        tg, tb = _grad_target(ctx.gamma), _grad_target(ctx.beta)
        gg = gb = None
        if tg is None:
            gg = tg = torch.zeros(ctx.c, dtype=torch.float32, device=dy.device)
        if tb is None:
            gb = tb = torch.zeros(ctx.c, dtype=torch.float32, device=dy.device)
        C_.layernorm_bwd(pre, dy, dx, ctx.gamma, mean, rstd, tg, tb, ctx.rows, ctx.c)
        return dx, (dx if ctx.has_res else None), gg, gb, None, None


class _AddLNFn(torch.autograd.Function):
    """Pre-LN residual step: ``s = x + residual`` and ``y = LN(s)``, both returned.  Backward takes ``dy`` and the skip
    gradient ``ds`` and writes ``dsum = LN_bwd(dy) + ds`` once, the gradient of both summands (no separate add)."""

    @staticmethod
    def forward(ctx, x, residual, gamma, beta, eps, anchor):
        gamma, beta = _unwrap(gamma), _unwrap(beta)
        c = x.shape[-1]
        rows = x.numel() // c
        y = torch.empty_like(x)
        s = torch.empty_like(x)
        mean = torch.empty(rows, dtype=torch.float32, device=x.device)
        rstd = torch.empty(rows, dtype=torch.float32, device=x.device)
        load().layernorm_sum_fwd(x, residual, y, s, gamma, beta, mean, rstd, rows, c, eps)
        ctx.save_for_backward(s, mean, rstd)
        ctx.set_materialize_grads(False)
        ctx.gamma, ctx.beta, ctx.rows, ctx.c = gamma, beta, rows, c
        return y, s

    @staticmethod
    def backward(ctx, dy, ds):
        s, mean, rstd = ctx.saved_tensors
        if dy is None:
            return ds, ds, None, None, None, None
        dy = dy.contiguous()
        dsum = torch.empty_like(s)
        tg, tb = _grad_target(ctx.gamma), _grad_target(ctx.beta)
        gg = gb = None
        if tg is None:
            gg = tg = torch.zeros(ctx.c, dtype=torch.float32, device=dy.device)
        if tb is None:
            gb = tb = torch.zeros(ctx.c, dtype=torch.float32, device=dy.device)
        if ds is None:       # the sum feeds nothing else (the last block's)
            load().layernorm_bwd(s, dy, dsum, ctx.gamma, mean, rstd, tg, tb, ctx.rows, ctx.c)
        else:
            load().layernorm_sum_bwd(s, dy, ds.contiguous(), dsum, ctx.gamma, mean, rstd, tg, tb, ctx.rows, ctx.c)
        return dsum, dsum, gg, gb, None, None


class _LNDropFn(torch.autograd.Function):
    """LayerNorm with dropout (csrc/dropout.cu).  mode 1, input dropout: ``LN(drop(x) + residual)``, the kernel writes
    the pre-norm sum; backward writes its gradient (the residual's) and ``M s`` times it (x's) in one launch.  mode 2,
    output dropout: ``drop(LN(x + residual))``; backward masks ``dy`` as it loads it.  ``dargs``: the dropout arguments
    of the kernel entry points (``DropoutRun.kernel_args``)."""

    @staticmethod
    def forward(ctx, x, residual, gamma, beta, eps, mode, dargs, anchor):
        gamma, beta = _unwrap(gamma), _unwrap(beta)
        c = x.shape[-1]
        rows = x.numel() // c
        y = torch.empty_like(x)
        mean = torch.empty(rows, dtype=torch.float32, device=x.device)
        rstd = torch.empty(rows, dtype=torch.float32, device=x.device)
        pre = torch.empty_like(x) if mode == 1 else None
        load().layernorm_drop_fwd(x, residual, y, pre, gamma, beta, mean, rstd, rows, c, eps, mode, *dargs)
        if mode == 2:
            pre = x if residual is None else F.add(x, residual)
        ctx.save_for_backward(pre, mean, rstd)
        ctx.gamma, ctx.beta, ctx.has_res, ctx.rows, ctx.c = gamma, beta, residual is not None, rows, c
        ctx.mode, ctx.dargs = mode, dargs
        return y

    @staticmethod
    def backward(ctx, dy):
        pre, mean, rstd = ctx.saved_tensors
        dy = dy.contiguous()
        dpre = torch.empty_like(pre)
        dx = torch.empty_like(pre) if ctx.mode == 1 else None
        tg, tb = _grad_target(ctx.gamma), _grad_target(ctx.beta)
        gg = gb = None
        if tg is None:
            gg = tg = torch.zeros(ctx.c, dtype=torch.float32, device=dy.device)
        if tb is None:
            gb = tb = torch.zeros(ctx.c, dtype=torch.float32, device=dy.device)
        load().layernorm_drop_bwd(pre, dy, dpre, dx, ctx.gamma, mean, rstd, tg, tb, ctx.rows, ctx.c, ctx.mode, *ctx.dargs)
        if ctx.mode == 2:
            dx = dpre
        return dx, (dpre if ctx.has_res else None), gg, gb, None, None, None, None


class LayerNorm(nn.Module):
    """``LN(x + residual)`` over the last axis (residual optional).  ``drop = (run, site, p, mode)``: the dropout form
    (``data/dropout.py``), mode 1 ``LN(drop(x) + residual)``, mode 2 ``drop(LN(x + residual))``."""

    def __init__(self, normalized_shape: int, eps: float = 1e-12):
        super().__init__()
        self.c, self.eps = normalized_shape, eps
        self.weight = nn.Parameter(torch.ones(normalized_shape))
        self.bias = nn.Parameter(torch.zeros(normalized_shape))

    def forward(self, x, residual=None, drop=None):
        if drop is not None:
            run, site, p, mode = drop
            if not x.is_cuda:
                if mode == 1:
                    x = run.apply(x, site, p)
                y = self.forward(x, residual)
                return run.apply(y, site, p) if mode == 2 else y
            return _LNDropFn.apply(x.contiguous(), None if residual is None else residual.contiguous(),
                                   _wrap(self.weight, x), _wrap(self.bias, x), self.eps, mode,
                                   run.kernel_args(site, p), _anchor(x, self.weight))
        if not x.is_cuda:
            if residual is not None:
                x = x + residual
            return TF.layer_norm(x, (self.c,), self.weight.to(x.dtype), self.bias.to(x.dtype), self.eps)
        return _LNFn.apply(x.contiguous(), None if residual is None else residual.contiguous(),
                           _wrap(self.weight, x), _wrap(self.bias, x), self.eps, _anchor(x, self.weight))

    def add_norm(self, x, residual):
        """``(LN(s), s)`` with ``s = x + residual``: the residual step of a pre-LN transformer block, which needs the sum
        as the next skip input.  On CUDA ``s`` is rounded to bf16 once and normalised as stored."""
        if not x.is_cuda:
            s = x + residual
            return TF.layer_norm(s, (self.c,), self.weight.to(s.dtype), self.bias.to(s.dtype), self.eps), s
        return _AddLNFn.apply(x.contiguous(), residual.contiguous(), _wrap(self.weight, x), _wrap(self.bias, x),
                              self.eps, _anchor(x, self.weight))


class _SoftmaxFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, scale):
        c = x.shape[-1]
        y = torch.empty_like(x)
        load().softmax_fwd(x, y, x.numel() // c, c, scale)
        ctx.save_for_backward(y)
        ctx.scale = scale
        return y

    @staticmethod
    def backward(ctx, dy):
        (y,) = ctx.saved_tensors
        c = y.shape[-1]
        dx = torch.empty_like(y)
        load().softmax_bwd(y, dy.contiguous(), dx, y.numel() // c, c, ctx.scale)
        return dx, None


def softmax(x: torch.Tensor, scale: float = 1.0) -> torch.Tensor:
    """``softmax(scale * x)`` over the last axis."""
    if not x.is_cuda:
        return torch.softmax(x * scale, dim=-1)
    return _SoftmaxFn.apply(x.contiguous(), scale)


# ================================================================================ losses
class _XentFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, logits, target, mix_row=None, smoothing=0.0):
        acc, dl = F.softmax_xent(logits, target, want_grad=True, mix_row=mix_row, smoothing=smoothing)
        ctx.save_for_backward(dl)
        ctx.mark_non_differentiable(acc)
        return acc[0].clone(), acc

    @staticmethod
    def backward(ctx, g, _unused):
        (dl,) = ctx.saved_tensors
        return dl * g.to(dl.dtype), None, None, None


def cross_entropy(logits: torch.Tensor, target: torch.Tensor, mix=None):
    """Fused softmax + NLL + gradient.  Returns ``(loss, stats)`` with
    ``stats = [mean loss, #correct]`` on the device.  ``mix = (mix_row, smoothing)``: the soft target of
    ``data/mix.py`` (``mix_row`` None: label smoothing only); the hits are then lam-weighted."""
    if not logits.is_cuda:
        if mix is not None:
            from ..data.mix import SoftTarget, decode_row, soft_cross_entropy, soft_hits
            row, eps = mix
            r = decode_row(row) if row is not None else None
            t = SoftTarget(target, target.roll(1, 0) if r else target, r.lam if r else 1.0, r.lam1 if r else 0.0, eps)
            loss = soft_cross_entropy(logits, t)
            return loss, torch.stack([loss.detach(), soft_hits(logits, t)])
        loss = TF.cross_entropy(logits.float(), target)
        hits = (logits.argmax(-1) == target).sum().float()
        return loss, torch.stack([loss.detach(), hits])
    if mix is not None:
        return _XentFn.apply(logits.contiguous(), target, mix[0], float(mix[1]))
    return _XentFn.apply(logits.contiguous(), target)


class _MseFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, pred, target):
        acc, dp = F.mse(pred, target, want_grad=True)
        ctx.save_for_backward(dp)
        return acc[0].clone()

    @staticmethod
    def backward(ctx, g):
        (dp,) = ctx.saved_tensors
        return dp * g.to(dp.dtype), None


def mse_loss(pred: torch.Tensor, target: torch.Tensor) -> torch.Tensor:
    if not pred.is_cuda:
        return TF.mse_loss(pred.float(), target.float().reshape(pred.shape))
    return _MseFn.apply(pred.contiguous(), target.reshape(pred.shape))


# ================================================================================ attention / embedding (BERT)
class _AttnFn(torch.autograd.Function):
    """Multi-head self-attention core on a packed ``qkv [B*S, 3*H*dh]`` buffer: four strided-batched
    wgmma GEMMs + the row-softmax kernel forward, five GEMMs + softmax backward; Q/K/V and their
    gradients are addressed in place through 4-D TMA maps (no head split / merge copies)."""

    @staticmethod
    def forward(ctx, qkv, B, S, H, dh, mask_bias=None, dargs=None):
        D = H * dh
        ctx.dargs = dargs
        ctx.short = S % 8 != 0
        if ctx.short:
            # S < 128 and not a multiple of 8 (ViT: patches + class token): the fused kernels with the tensor dimension S,
            # probs [B*H, S, round_up(S, 8)]
            if not (S < 128 and dh == 64 and mask_bias is None and dargs is None):
                raise ValueError("attention: S = {} is not a multiple of 8, which only the fused kernel for S < 128, "
                                 "d_head = 64 without mask or dropout runs (got d_head = {}{}{})".format(
                                     S, dh, ", a mask" if mask_bias is not None else "",
                                     ", dropout" if dargs is not None else ""))
            probs = torch.empty((B * H, S, (S + 7) // 8 * 8), dtype=BF16, device=qkv.device)
            out = torch.empty((B * S, D), dtype=BF16, device=qkv.device)
            load().attention_short_fwd(qkv, out, probs, B, S, H, dh, 1.0 / math.sqrt(dh))
            ctx.save_for_backward(qkv, probs, None)
            ctx.dims = (B, S, H, dh)
            return out
        if S == 128 and dh == 64 and mask_bias is None:
            # single-kernel forward (csrc/attention.cu): scores stay in shared memory, P is written once
            probs = torch.empty((B * H * S, S), dtype=BF16, device=qkv.device)
            out = torch.empty((B * S, D), dtype=BF16, device=qkv.device)
            ok = (load().attention_fwd(qkv, out, probs, B, S, H, dh, 1.0 / math.sqrt(dh)) if dargs is None else
                  load().attention_drop_fwd(qkv, out, probs, B, S, H, dh, 1.0 / math.sqrt(dh), *dargs))
            if ok:
                ctx.save_for_backward(qkv, probs, None)
                ctx.dims = (B, S, H, dh)
                return out
        q, k, v = qkv[:, :D], qkv[:, D:2 * D], qkv[:, 2 * D:]
        scores = torch.empty((B * H * S, S), dtype=BF16, device=qkv.device)
        F.gemm_batched(q, k, scores, M=S, N=S, K=dh, lda=3 * D, ldb=3 * D, ldd=S, a_mn=False, b_mn=False,
                       n_outer=B, n_inner=H, a_strides=(S * 3 * D, dh), b_strides=(S * 3 * D, dh),
                       d_strides=(H * S * S, S * S), alpha=1.0 / math.sqrt(dh))
        if mask_bias is not None:        # additive key-padding mask [B, S] (0 / large negative), broadcast over heads and queries
            scores.view(B, H, S, S).add_(mask_bias.to(scores.dtype).view(B, 1, 1, S))
        probs = torch.empty_like(scores)
        pdrop = None
        if dargs is None:
            load().softmax_fwd(scores, probs, B * H * S, S, 1.0)
        else:        # P is saved for backward, the dropped P (the one extra S x S buffer) feeds the PV GEMM and dV
            pdrop = torch.empty_like(scores)
            load().softmax_drop_fwd(scores, probs, pdrop, B * H * S, S, 1.0, *dargs)
        out = torch.empty((B * S, D), dtype=BF16, device=qkv.device)
        F.gemm_batched(probs if pdrop is None else pdrop, v, out, M=S, N=dh, K=S, lda=S, ldb=3 * D, ldd=D, a_mn=False, b_mn=True,
                       n_outer=B, n_inner=H, a_strides=(H * S * S, S * S), b_strides=(S * 3 * D, dh),
                       d_strides=(S * D, dh))
        ctx.save_for_backward(qkv, probs, pdrop)
        ctx.dims = (B, S, H, dh)
        ctx.masked = mask_bias is not None
        return out

    @staticmethod
    def backward(ctx, dout):
        qkv, probs, pdrop = ctx.saved_tensors
        B, S, H, dh = ctx.dims
        D = H * dh
        dargs = ctx.dargs
        dout = dout.contiguous()
        dqkv = torch.empty_like(qkv)
        if ctx.short:
            load().attention_short_bwd(qkv, dout, probs, dqkv, B, S, H, dh, 1.0 / math.sqrt(dh))
            return dqkv, None, None, None, None, None, None
        if S == 128 and dh == 64 and not getattr(ctx, "masked", False):
            # single-kernel backward (csrc/attention.cu): dP / dS never leave the SM
            ok = (load().attention_bwd(qkv, dout, probs, dqkv, B, S, H, dh, 1.0 / math.sqrt(dh)) if dargs is None else
                  load().attention_drop_bwd(qkv, dout, probs, dqkv, B, S, H, dh, 1.0 / math.sqrt(dh), *dargs))
            if ok:
                return dqkv, None, None, None, None, None, None
        q, k, v = qkv[:, :D], qkv[:, D:2 * D], qkv[:, 2 * D:]
        dq, dk, dv = dqkv[:, :D], dqkv[:, D:2 * D], dqkv[:, 2 * D:]
        bh = (H * S * S, S * S)
        pk = (S * 3 * D, dh)
        # dV = P^T dO (the dropped P with dropout)
        F.gemm_batched(probs if pdrop is None else pdrop, dout, dv, M=S, N=dh, K=S, lda=S, ldb=D, ldd=3 * D, a_mn=True, b_mn=True,
                       n_outer=B, n_inner=H, a_strides=bh, b_strides=(S * D, dh), d_strides=pk)
        # dP = dO V^T
        dprobs = torch.empty_like(probs)
        F.gemm_batched(dout, v, dprobs, M=S, N=S, K=dh, lda=D, ldb=3 * D, ldd=S, a_mn=False, b_mn=False,
                       n_outer=B, n_inner=H, a_strides=(S * D, dh), b_strides=pk, d_strides=bh)
        dscores = torch.empty_like(probs)
        if dargs is None:
            load().softmax_bwd(probs, dprobs, dscores, B * H * S, S, 1.0)
        else:
            load().softmax_drop_bwd(probs, dprobs, dscores, B * H * S, S, 1.0, *dargs)
        alpha = 1.0 / math.sqrt(dh)
        # dQ = alpha dS K ; dK = alpha dS^T Q
        F.gemm_batched(dscores, k, dq, M=S, N=dh, K=S, lda=S, ldb=3 * D, ldd=3 * D, a_mn=False, b_mn=True,
                       n_outer=B, n_inner=H, a_strides=bh, b_strides=pk, d_strides=pk, alpha=alpha)
        F.gemm_batched(dscores, q, dk, M=S, N=dh, K=S, lda=S, ldb=3 * D, ldd=3 * D, a_mn=True, b_mn=True,
                       n_outer=B, n_inner=H, a_strides=bh, b_strides=pk, d_strides=pk, alpha=alpha)
        return dqkv, None, None, None, None, None, None


def attention(qkv: torch.Tensor, B: int, S: int, H: int, dh: int, mask_bias: Optional[torch.Tensor] = None,
              drop=None) -> torch.Tensor:
    """``softmax(Q K^T / sqrt(dh) + mask_bias) V`` for packed ``qkv [B*S, 3*H*dh]`` -> ``[B*S, H*dh]``.
    ``mask_bias``: optional additive key mask ``[B, S]`` (0 = attend, large negative = padding).  ``drop = (run, site,
    p)``: dropout on the probabilities (``data/dropout.py``), element i the index into ``[B*H*S, S]``."""
    if not qkv.is_cuda:
        D = H * dh
        q, k, v = (t.reshape(B, S, H, dh).transpose(1, 2) for t in qkv.split(D, dim=-1))
        sc = q @ k.transpose(-1, -2) / math.sqrt(dh)
        if mask_bias is not None:
            sc = sc + mask_bias.to(sc.dtype).view(B, 1, 1, S)
        p = torch.softmax(sc, dim=-1)
        if drop is not None:
            run, site, pr = drop
            p = run.apply(p.contiguous(), site, pr)
        return (p @ v).transpose(1, 2).reshape(B * S, D)
    dargs = drop[0].kernel_args(drop[1], drop[2]) if drop is not None else None
    return _AttnFn.apply(qkv.contiguous(), B, S, H, dh, mask_bias, dargs)


class _TokensFn(torch.autograd.Function):
    """ViT token assembly (csrc/elementwise.cu): forward one launch, backward one launch that writes the patch gradient
    and accumulates the class-token, bias and position-embedding gradients in a fixed order."""

    @staticmethod
    def forward(ctx, z, cls, bias, pos, anchor):
        cls, bias, pos = _unwrap(cls), _unwrap(bias), _unwrap(pos)
        B, N, D = z.shape
        tok = torch.empty((B, N + 1, D), dtype=BF16, device=z.device)
        load().vit_tokens_fwd(z, cls.detach(), bias.detach(), pos.detach(), tok, B, N + 1, D)
        ctx.params = (cls, bias, pos)
        return tok

    @staticmethod
    def backward(ctx, dtok):
        B, S, D = dtok.shape
        tgts, grads = [], []
        for p in ctx.params:
            t = _grad_target(p)
            g = None
            if t is None:
                g = t = torch.zeros_like(p, dtype=torch.float32)
            tgts.append(t)
            grads.append(g)
        dz = torch.empty((B, S - 1, D), dtype=BF16, device=dtok.device)
        load().vit_tokens_bwd(dtok.contiguous(), dz, *tgts, B, S, D)
        return (dz, *grads, None)


def vit_tokens(z: torch.Tensor, cls: torch.Tensor, bias: torch.Tensor, pos: torch.Tensor) -> torch.Tensor:
    """``[cls; z + bias] + pos``: the token sequence ``[B, 1 + N, D]`` of a Vision Transformer from its patch embeddings
    ``z [B, N, D]`` (without the projection bias), the class token ``[1, 1, D]``, the projection bias ``[D]`` and the
    position embedding ``[1, 1 + N, D]``.  On CUDA each token is summed in fp32 and rounded to bf16 once."""
    if not z.is_cuda:
        B = z.shape[0]
        return torch.cat([cls.to(z.dtype).expand(B, -1, -1), z + bias.to(z.dtype)], dim=1) + pos.to(z.dtype)
    return _TokensFn.apply(z.contiguous(), _wrap(cls, z), _wrap(bias, z), _wrap(pos, z), _anchor(z, cls, bias, pos))


class _DropFn(torch.autograd.Function):
    """Elementwise dropout of a bf16 tensor (``csrc/dropout.cu``): forward and backward apply the same mask."""

    @staticmethod
    def forward(ctx, x, dargs):
        y = torch.empty_like(x)
        load().dropout(x, y, *dargs)
        ctx.dargs = dargs
        return y

    @staticmethod
    def backward(ctx, dy):
        dx = torch.empty_like(dy, memory_format=torch.contiguous_format)
        load().dropout(dy.contiguous(), dx, *ctx.dargs)
        return dx, None


def dropout(x: torch.Tensor, run, site: int, p: float) -> torch.Tensor:
    """``x`` with the mask of dropout ``site`` at ``run``'s current step (``data/dropout.py``)."""
    if not x.is_cuda:
        return run.apply(x, site, p)
    if x.dtype != BF16:
        x = F.cast(x.contiguous(), BF16)
    return _DropFn.apply(x.contiguous(), run.kernel_args(site, p))


class _EmbedFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, table, table_bf16, ids, anchor):
        table = _unwrap(table)
        ctx.save_for_backward(ids)
        ctx.table = table
        return F.gather_rows(table_bf16, ids)

    @staticmethod
    def backward(ctx, dy):
        (ids,) = ctx.saved_tensors
        table = ctx.table
        if _frozen(table):
            return None, None, None, None
        tgt = _grad_target(table)
        g = None
        if tgt is None:
            g = tgt = torch.zeros_like(table, dtype=torch.float32)
        F.embedding_bwd_(dy.contiguous(), ids, tgt)
        return g, None, None, None


class Embedding(nn.Module):
    """Lookup in the bf16 shadow of an fp32 table; gradient scattered with fp32 atomics."""

    def __init__(self, num_embeddings: int, embedding_dim: int):
        super().__init__()
        self.weight = nn.Parameter(torch.randn(num_embeddings, embedding_dim) * 0.02)

    def forward(self, ids):
        flat = ids.reshape(-1)
        if not ids.is_cuda:
            return TF.embedding(flat, self.weight)
        return _EmbedFn.apply(_wrap(self.weight, flat), _shadow(self, "weight", self.weight), flat,
                              _anchor(flat, self.weight))


# ================================================================================ MXFP8 matmul (block-scaled fp8 training)
class _MatmulFp8Fn(torch.autograd.Function):
    """``y = x w^T`` with every GEMM of the layer -- forward, dgrad, wgrad -- on the block-scaled
    fp8 tensor-core path.  Each operand is quantised (e4m3 + UE8M0 scale per 32 elements) along the
    reduction dimension of the GEMM that consumes it; the transposed operands of dgrad / wgrad come
    out of the fused quantise+transpose kernel, so the GEMM kernel only ever sees K-major inputs.
    The weight gradient is accumulated in fp32 straight into the gradient arena."""

    @staticmethod
    def forward(ctx, x2, weight, w_bf16, k_true, anchor):
        weight = _unwrap(weight)
        K = x2.shape[1]
        xq, sx = F.quant_mx_rows(x2)
        wq, sw = F.quant_mx_rows(w_bf16)
        y = F.gemm_fp8(xq, sx, wq, sw, K)
        ctx.save_for_backward(x2, w_bf16)
        ctx.weight, ctx.k_true = weight, k_true
        ctx.needs_dx = x2.requires_grad
        return y

    @staticmethod
    def backward(ctx, dy):
        x2, w_bf16 = ctx.saved_tensors
        dy = dy.contiguous()
        M, N = dy.shape
        K = x2.shape[1]
        weight, k_true = ctx.weight, ctx.k_true
        # wgrad: dW[N, K] = dY^T[N, M] X^T[K, M]^T   (reduction over M)
        dyt, sdyt = F.quant_mx_cols(dy)
        xt, sxt = F.quant_mx_cols(x2)
        gw = None
        tgt = _grad_target(weight)
        if tgt is not None:
            out2d = tgt.permute(0, 2, 3, 1).reshape(N, k_true) if tgt.dim() == 4 else tgt.view(N, k_true)
            F.gemm_fp8(dyt, sdyt, xt, sxt, M, out=out2d, accumulate=True, n_valid=k_true)
        else:
            g2 = F.gemm_fp8(dyt, sdyt, xt, sxt, M, out_dtype=torch.float32, accumulate=True, n_valid=k_true)
            gw = g2.view(weight.shape[0], *weight.shape[2:], weight.shape[1]).permute(0, 3, 1, 2) if weight.dim() == 4 \
                else g2.view_as(weight)
        dx = None
        if ctx.needs_dx:
            # dgrad: dX[M, K] = dY[M, N] (W^T)[K, N]^T   (reduction over N)
            dyq, sdy = F.quant_mx_rows(dy)
            wt, swt = F.quant_mx_cols(w_bf16)
            dx = F.gemm_fp8(dyq, sdy, wt, swt, N)
        return dx, gw, None, None, None


def matmul_fp8(x2: torch.Tensor, module: nn.Module, w_bf16: torch.Tensor, k_true: int) -> torch.Tensor:
    return _MatmulFp8Fn.apply(x2, _wrap(module.weight, x2), w_bf16, k_true, _anchor(x2, module.weight))


class _Im2colFn(torch.autograd.Function):
    """im2col as its own differentiable op (its adjoint is col2im) so the fp8 matmul above can sit
    between it and the BatchNorm that follows."""

    @staticmethod
    def forward(ctx, x, kh, kw, stride, pad):
        col, ho, wo, kp = F.im2col(x, kh, kw, stride, pad)
        ctx.geom = (tuple(x.shape), kh, kw, stride, pad, ho, wo)
        return col

    @staticmethod
    def backward(ctx, dcol):
        shape, kh, kw, stride, pad, ho, wo = ctx.geom
        return F.col2im(dcol.contiguous(), shape, kh, kw, stride, pad, ho, wo), None, None, None, None


def conv2d_fp8(x: torch.Tensor, conv: "Conv2d") -> torch.Tensor:
    """NHWC convolution with all three GEMMs in MXFP8."""
    n, h, w, c = x.shape
    k, s, p = conv.kernel_size, conv.stride, conv.padding
    ho, wo = F.conv_out_size(h, k, s, p), F.conv_out_size(w, k, s, p)
    if k == 1 and s == 1 and p == 0 and c % 16 == 0:
        col = x.reshape(n * h * w, c)
    elif c % 8 == 0:
        col = _Im2colFn.apply(x, k, k, s, p)
    else:   # stem (C = 3): no input gradient needed, plain im2col
        col = F.im2col(x, k, k, s, p)[0]
    y = matmul_fp8(col, conv, conv._w_bf16(), conv.k_true)
    return y.view(n, ho, wo, conv.out_channels)
