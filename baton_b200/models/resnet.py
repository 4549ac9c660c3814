"""ResNet-18 / ResNet-50 on the sm_90a layers.

Architecture and ``state_dict`` keys follow the standard ImageNet-style ResNet
(7x7/2 stem, 3x3/2 max-pool, four stages, global average pool, linear head), so
a stock PyTorch ResNet ``state_dict`` of the same depth loads unchanged -- the
"checkpoint layout stays compatible" requirement.  With ``num_classes=10`` the
ResNet-18 float state is 11,191,242 elements (SURVEY.md section 5.1).

Execution differs from a stock model: activations are bf16 NHWC, every
convolution is a wgmma GEMM (implicit GEMM over TMA im2col loads where the
shape allows it, explicit im2col otherwise), BatchNorm fuses the residual add
and the ReLU of the block, parameters live in the flat arena.  The user-model contract
(``name``, ``__hash__``, ``train(X, y, n_epoch=...)``) comes from
``FederatedModule`` (reference demo.py:15-49).
"""
from __future__ import annotations

from typing import List, Optional, Sequence, Type

import torch
from torch import nn

from ..ops import nn as bnn
from .base import FederatedModule


# ---------------------------------------------------------------------------------------------------------------
# Hand-scheduled training step (no autograd engine).  The layer kernels are the ones the autograd Functions in
# ``ops/nn.py`` call -- their ``forward`` / ``backward`` bodies are driven directly through ``bnn.Ctx`` -- but the
# schedule is ours: the gradient of a block input travels as TWO pieces (main-branch dgrad, residual-branch
# gradient) that the consuming BatchNorm-backward kernel sums while loading, so the eight element-wise adds autograd
# would launch per step disappear; the downsample branch runs as a parallel branch of the captured graph.
# ---------------------------------------------------------------------------------------------------------------
def _conv_bn_fwd(conv: "bnn.Conv2d", bn: "bnn.BatchNorm2d", x, residual=None, after_conv=None):
    cc, cb = bnn.Ctx(), bnn.Ctx()
    stats = conv._fusable_stats(x)
    z = bnn._ConvFn.forward(cc, x, conv.weight, conv._w_bf16(), conv.plan(x), None, stats, conv.flags_cfg)
    if after_conv is not None:
        after_conv()
    y = bnn._BNFn.forward(cb, z, residual, bn.weight, bn.bias, bn.running_mean, bn.running_var, bn.num_batches_tracked,
                          bn.eps, bn.momentum, bn.relu, True, bn.workspace, None, stats is not None)
    return y, (cc, cb)


def _conv_bn_bwd(ctxs, dy_a, dy_b=None, needs_dx=True):
    """-> (gradient w.r.t. the conv input, gradient w.r.t. the residual input or None)"""
    cc, cb = ctxs
    cc.needs_dx = needs_dx
    out = bnn._BNFn.backward(cb, dy_a, dy_b)
    dz, dres = out[0], out[1]
    dx = bnn._ConvFn.backward(cc, dz)[0]
    return dx, dres


# The same pair for GroupNorm: the conv GEMM takes no statistics (they are per sample, computed by gn_fwd itself).
def _conv_gn_fwd(conv: "bnn.Conv2d", gn: "bnn.GroupNorm", x, residual=None, after_conv=None):
    cc, cg = bnn.Ctx(), bnn.Ctx()
    z = bnn._ConvFn.forward(cc, x, conv.weight, conv._w_bf16(), conv.plan(x), None, None, conv.flags_cfg)
    if after_conv is not None:
        after_conv()
    y = bnn._GNFn.forward(cg, z, residual, gn.weight, gn.bias, gn.num_groups, gn.eps, gn.relu, True, None)
    return y, (cc, cg)


def _conv_gn_bwd(ctxs, dy_a, dy_b=None, needs_dx=True):
    cc, cg = ctxs
    cc.needs_dx = needs_dx
    dz, dres = bnn._GNFn.backward(cg, dy_a, dy_b)[:2]
    dx = bnn._ConvFn.backward(cc, dz)[0]
    return dx, dres


_CONV_NORM = {"batch": (_conv_bn_fwd, _conv_bn_bwd), "group": (_conv_gn_fwd, _conv_gn_bwd)}


# The stem (conv1 -> bn1 -> relu -> maxpool): BatchNorm + ReLU + max-pool are ONE kernel forward and two backward (the
# normalised 16x16 activation is never written: the pooled output carries the ReLU mask, BatchNorm's backward sums run
# over the pooled gradient -- csrc/norm.cu, "ResNet stem").  Where _stem_fwd declines, the separate kernels run.


def _stem_fwd(conv, bn, pool, x, after_conv=None):
    """-> ``(pooled, conv ctx, z, argmax, mean, rstd)`` or ``None`` when the fused kernels do not apply."""
    stats = conv._fusable_stats(x)
    if (stats is None or bn.workspace is None or not bn.relu or not bn.training or bn.num_features % 8
            or bnn._grad_target(bn.weight) is None or bnn._grad_target(bn.bias) is None):
        return None
    cc = bnn.Ctx()
    z = bnn._ConvFn.forward(cc, x, conv.weight, conv._w_bf16(), conv.plan(x), None, stats, conv.flags_cfg)
    if after_conv is not None:
        after_conv()
    c = bn.num_features
    out = bnn.F.bn_relu_maxpool(z, bn.workspace[: 2 * c], bnn._unwrap(bn.weight), bnn._unwrap(bn.bias), bn.running_mean,
                                bn.running_var, bn.num_batches_tracked, bn.eps, bn.momentum, pool.k, pool.stride, pool.pad)
    if out is None:
        raise RuntimeError("bn_relu_maxpool rejected a shape _stem_fwd accepted")
    p, arg, mean, rstd = out
    return p, cc, z, arg, mean, rstd


def _stem_bwd(saved, bn, pool, dy_a, dy_b=None):
    p, cc, z, arg, mean, rstd = saved
    c = bn.num_features
    gamma = bnn._unwrap(bn.weight)
    tg, tb = bnn._grad_target(gamma), bnn._grad_target(bnn._unwrap(bn.bias))
    dz = bnn.F.bn_maxpool_bwd(z, p, arg, dy_a.contiguous(), dy_b.contiguous() if dy_b is not None else None, gamma, mean,
                              rstd, bn.workspace[2 * c:], tg, tb, pool.k, pool.stride, pool.pad)
    if dz is None:
        raise RuntimeError("bn_maxpool_bwd rejected a shape bn_relu_maxpool accepted")
    cc.needs_dx = False
    bnn._ConvFn.backward(cc, dz)


# Evaluation (``ResNet.explicit_eval``): every conv + BatchNorm pair is ONE GEMM whose epilogue applies the eval-mode
# BatchNorm -- the per-channel scale / shift that ``F.bn_fold_eval`` wrote into ``model.eval_bn_table`` at the
# BatchNorm's ``eval_off`` -- plus the block's shortcut and the ReLU.  Where a GEMM declines the epilogue, the plain
# GEMM and ``bn_apply(training=0)`` run instead.  The bf16 weights come from ``ResNet.prepare_eval`` (once per pass).
def _conv_bn_eval(conv, bn, x, table, residual=None):
    plan, wt = conv.plan(x), conv.eval_weight
    af = bnn.F.affine_epilogue_args(table, bn.eval_off, plan.cout, bn.relu, residual)
    y = bnn.F.conv_fwd(x, wt, plan, affine=af)[0]
    if y is None:
        z = bnn._ConvFn.forward(bnn.Ctx(), x, conv.weight, wt, plan, None)
        y = bnn._BNFn.forward(bnn.Ctx(), z, residual, bn.weight, bn.bias, bn.running_mean, bn.running_var, None, bn.eps,
                              bn.momentum, bn.relu, False, None, None)
    return y.view(plan.n, plan.ho, plan.wo, plan.cout)


def _batch_norm(c: int, relu: bool) -> nn.Module:
    return bnn.BatchNorm2d(c, relu=relu)


def _group_norm(groups: int):
    return lambda c, relu: bnn.GroupNorm(groups, c, relu=relu)


class BasicBlock(nn.Module):
    expansion = 1

    def __init__(self, inplanes: int, planes: int, stride: int = 1, downsample: Optional[nn.Module] = None,
                 norm=_batch_norm):
        super().__init__()
        self.conv1 = bnn.Conv2d(inplanes, planes, 3, stride, 1)
        self.bn1 = norm(planes, True)
        self.conv2 = bnn.Conv2d(planes, planes, 3, 1, 1)
        self.bn2 = norm(planes, True)                       # relu(bn2(.) + identity), fused
        self.downsample = downsample

    def forward(self, x):
        identity = x if self.downsample is None else self.downsample(x)
        out = self.bn1(self.conv1(x))
        return self.bn2(self.conv2(out), identity)

    units = (("conv1", "bn1"), ("conv2", "bn2"))


class Bottleneck(nn.Module):
    expansion = 4

    def __init__(self, inplanes: int, planes: int, stride: int = 1, downsample: Optional[nn.Module] = None,
                 norm=_batch_norm):
        super().__init__()
        self.conv1 = bnn.Conv2d(inplanes, planes, 1, 1, 0)
        self.bn1 = norm(planes, True)
        self.conv2 = bnn.Conv2d(planes, planes, 3, stride, 1)
        self.bn2 = norm(planes, True)
        self.conv3 = bnn.Conv2d(planes, planes * 4, 1, 1, 0)
        self.bn3 = norm(planes * 4, True)
        self.downsample = downsample

    def forward(self, x):
        identity = x if self.downsample is None else self.downsample(x)
        out = self.bn1(self.conv1(x))
        out = self.bn2(self.conv2(out))
        return self.bn3(self.conv3(out), identity)

    units = (("conv1", "bn1"), ("conv2", "bn2"), ("conv3", "bn3"))


class _Downsample(nn.Sequential):
    """``0`` = 1x1 strided conv, ``1`` = BatchNorm or GroupNorm (same indices as the stock model)."""

    def __init__(self, inplanes: int, outplanes: int, stride: int, norm=_batch_norm):
        super().__init__(bnn.Conv2d(inplanes, outplanes, 1, stride, 0), norm(outplanes, False))


class ResNet(FederatedModule):
    loss_kind = "ce"
    default_lr = 0.05
    default_batch_size = 128
    head = "fc"
    # read by ParamArena: the hand-scheduled step applies the optimizer in the convolution weight-gradient epilogues
    frozen_params_unsupported = ("ResNets do not support frozen parameters: their hand-scheduled training step "
                                 "(explicit_step) computes and applies a gradient for every convolution, BatchNorm and "
                                 "fc parameter")

    def __init__(self, block: Type[nn.Module], layers: Sequence[int], num_classes: int = 1000,
                 in_channels: int = 3, name: Optional[str] = None, norm: str = "batch", groups: int = 2):
        """``norm="group"``: every BatchNorm becomes a ``GroupNorm(groups, C)`` under the same name (torchvision's model
        built with ``norm_layer=lambda c: nn.GroupNorm(groups, c)``), so the model has no buffers."""
        super().__init__()
        if norm not in _CONV_NORM:
            raise ValueError("ResNet: norm must be 'batch' or 'group', got {!r}".format(norm))
        if name:
            self.name = name
        self.norm = norm
        norm_layer = _batch_norm if norm == "batch" else _group_norm(groups)
        self.inplanes = 64
        self.conv1 = bnn.Conv2d(in_channels, 64, 7, 2, 3)
        self.bn1 = norm_layer(64, True)
        self.maxpool = bnn.MaxPool2d(3, 2, 1)
        self.layer1 = self._make_layer(block, 64, layers[0], 1, norm_layer)
        self.layer2 = self._make_layer(block, 128, layers[1], 2, norm_layer)
        self.layer3 = self._make_layer(block, 256, layers[2], 2, norm_layer)
        self.layer4 = self._make_layer(block, 512, layers[3], 2, norm_layer)
        self.avgpool = bnn.GlobalAvgPool()
        self.fc = bnn.Linear(512 * block.expansion, num_classes, out_fp32=True)
        self.stats_workspace = None
        self.zeroes_own_workspace = True   # forward() clears the statistics workspace itself
        for m in self.modules():   # zero-init the last BN of each block (standard recipe; keeps early training stable)
            if isinstance(m, BasicBlock):
                nn.init.zeros_(m.bn2.weight)
            elif isinstance(m, Bottleneck):
                nn.init.zeros_(m.bn3.weight)

    def _make_layer(self, block, planes: int, blocks: int, stride: int, norm_layer) -> nn.Sequential:
        downsample = None
        if stride != 1 or self.inplanes != planes * block.expansion:
            downsample = _Downsample(self.inplanes, planes * block.expansion, stride, norm_layer)
        layers: List[nn.Module] = [block(self.inplanes, planes, stride, downsample, norm_layer)]
        self.inplanes = planes * block.expansion
        for _ in range(1, blocks):
            layers.append(block(self.inplanes, planes, norm=norm_layer))
        return nn.Sequential(*layers)

    def set_precision(self, dtype: str = "bf16") -> "ResNet":
        """``"fp8"``: every convolution (forward, dgrad and wgrad GEMMs) runs on the block-scaled
        MXFP8 tensor-core path; BatchNorm, the classifier head and the optimizer stay bf16/fp32."""
        assert dtype in ("bf16", "fp8")
        for m in self.modules():
            if isinstance(m, bnn.Conv2d):
                m.fp8 = dtype == "fp8"
        self.compute_dtype = dtype
        return self

    def forward(self, x):
        """``x``: NHWC ``[N, H, W, C]`` (bf16 on CUDA)."""
        if self.stats_workspace is not None and self.training:
            self.stats_workspace.zero_()      # ONE memset per step: forward and backward statistic sums of every BN
        x = self.maxpool(self.bn1(self.conv1(x)))
        x = self.layer4(self.layer3(self.layer2(self.layer1(x))))
        return self.fc(self.avgpool(x))

    # ------------------------------------------------------------------ hand-scheduled step
    def _block_fwd(self, blk, x, tape):
        ds_ctx = None
        identity = x
        if blk.downsample is not None:
            with bnn.BRANCH.fork(x):                      # parallel graph branch: 1x1 conv + BN of the shortcut
                identity, ds_ctx = _CONV_NORM[self.norm][0](blk.downsample[0], blk.downsample[1], x)
        out = x
        ctxs = []
        n = len(blk.units)
        for i, (cn, bnn_) in enumerate(blk.units):
            last = i == n - 1
            if last:
                bnn.BRANCH.join()                         # the shortcut must have landed before the residual add
            out, c = _CONV_NORM[self.norm][0](getattr(blk, cn), getattr(blk, bnn_), out, identity if last else None)
            ctxs.append(c)
        tape.append((ctxs, ds_ctx))
        return out

    def _block_bwd(self, entry, pieces):
        """``pieces``: 1-2 tensors whose sum is the gradient of the block output -> pieces of the block-input gradient"""
        ctxs, ds_ctx = entry
        bwd = _CONV_NORM[self.norm][1]
        d, dres = bwd(ctxs[-1], pieces[0], pieces[1] if len(pieces) > 1 else None)
        dx_ds = None
        if ds_ctx is not None:
            with bnn.BRANCH.fork(dres):                   # shortcut backward in parallel with the main branch
                dx_ds, _ = bwd(ds_ctx, dres)
        for c in reversed(ctxs[:-1]):
            d, _ = bwd(c, d)
        if ds_ctx is not None:
            bnn.BRANCH.join()
            return [d, dx_ds]
        return [d, dres]

    def explicit_step(self, x, target, loss_acc=None, after_first_gemm=None, mix=None):
        """Forward + loss + backward of one batch with parameter gradients accumulated into the arena (the same
        contract as ``loss.backward()`` on ``forward``); returns the device ``[mean loss, #correct]`` pair.
        CUDA + arena-adopted training mode only.

        ``after_first_gemm`` (optional, from the trainer) is called right after the GEMM of the first convolution.
        ``mix = (mix_row, smoothing)``: the soft-target loss of ``data/mix.py`` in both head paths."""
        soft = dict(mix_row=mix[0], smoothing=float(mix[1])) if mix is not None else {}
        F = bnn.F
        if self.stats_workspace is not None:
            self.stats_workspace.zero_()
        stem = cp = None
        fwd, bwd = _CONV_NORM[self.norm]
        fused_stem = _stem_fwd(self.conv1, self.bn1, self.maxpool, x, after_first_gemm) if self.norm == "batch" else None
        if fused_stem is not None:
            h = fused_stem[0]
        else:
            h, stem = fwd(self.conv1, self.bn1, x, after_conv=after_first_gemm)
            cp = bnn.Ctx()
            h = bnn._MaxPoolFn.forward(cp, h, self.maxpool.k, self.maxpool.stride, self.maxpool.pad)
        tape = []
        for layer in (self.layer1, self.layer2, self.layer3, self.layer4):
            for blk in layer:
                h = self._block_fwd(blk, h, tape)
        ca = None
        if h.shape[1] == 1 and h.shape[2] == 1:
            feat = h.reshape(h.shape[0], h.shape[3])
        else:
            ca = bnn.Ctx()
            feat = bnn._AvgPoolFn.forward(ca, h)
        fc = self.fc
        head = None
        tw, tb = bnn._grad_target(fc.weight), bnn._grad_target(fc.bias)
        if fc.out_features <= 32 and tw is not None and (fc.bias is None or tb is not None) and fc.act == 0:
            # classifier head (linear + softmax cross-entropy, forward and backward) in ONE launch
            head = F.linear_xent_head(feat.contiguous(), bnn._shadow(fc, "weight", fc.weight), fc.bias, target, tw, tb,
                                      acc=loss_acc, **soft)
        if head is not None:
            stats, d, _ = head
        else:
            cl = bnn.Ctx()
            logits = bnn._LinearFn.forward(cl, feat, fc.weight, fc.bias, bnn._shadow(fc, "weight", fc.weight), fc.act,
                                           fc.out_fp32, None, None)
            cl.needs_dx = True
            stats, dlogits = F.softmax_xent(logits.contiguous(), target, want_grad=True, acc=loss_acc, **soft)
            d = bnn._LinearFn.backward(cl, dlogits)[0]
        d = d.reshape(h.shape) if ca is None else bnn._AvgPoolFn.backward(ca, d)
        pieces = [d]
        for bi in range(len(tape) - 1, -1, -1):
            pieces = self._block_bwd(tape[bi], pieces)
        if fused_stem is not None:
            _stem_bwd(fused_stem, self.bn1, self.maxpool, pieces[0], pieces[1] if len(pieces) > 1 else None)
        else:
            d = bnn._MaxPoolFn.backward(cp, pieces[0], pieces[1] if len(pieces) > 1 else None)[0]
            bwd(stem, d, needs_dx=False)
        bnn.WGRAD.join()
        return stats

    # ------------------------------------------------------------------ evaluation
    def _block_eval(self, blk, x, table):
        identity = x
        if blk.downsample is not None:
            with bnn.BRANCH.fork(x):                      # parallel graph branch: 1x1 conv + BN of the shortcut
                identity = _conv_bn_eval(blk.downsample[0], blk.downsample[1], x, table)
        out = x
        n = len(blk.units)
        for i, (cn, bn_name) in enumerate(blk.units):
            last = i == n - 1
            if last:
                bnn.BRANCH.join()
            out = _conv_bn_eval(getattr(blk, cn), getattr(blk, bn_name), out, table, identity if last else None)
        return out

    def prepare_eval(self):
        """Head of an evaluation pass: the bf16 weights every ``explicit_eval`` of the pass reads (the stem's
        zero-padded copy is made here, once, instead of per batch; the others are views of the arena shadow)."""
        for m in self.modules():
            if isinstance(m, bnn.Conv2d):
                m.eval_weight = m._w_bf16(gated=False)   # evaluation runs after the collective has been joined

    def explicit_eval(self, x, target, acc, want_logits: bool = False):
        """Forward-only pass of one batch in eval mode (running statistics): adds the SUM of the row cross-entropies
        and the number of correct predictions into ``acc`` (fp32 ``[2]``); returns the fp32 logits when
        ``want_logits``, else ``None``.  Every BatchNorm runs in the epilogue of its
        convolution GEMM, reading the scale / shift that ``F.bn_fold_eval`` wrote into ``self.eval_bn_table`` and the
        weights of :meth:`prepare_eval` (both run at the head of the pass).  Saves
        nothing for a backward pass and writes no model state.  CUDA, bf16 only."""
        F = bnn.F
        table = self.eval_bn_table
        h = _conv_bn_eval(self.conv1, self.bn1, x, table)
        h = F.maxpool(h, self.maxpool.k, self.maxpool.stride, self.maxpool.pad)[0]
        for layer in (self.layer1, self.layer2, self.layer3, self.layer4):
            for blk in layer:
                h = self._block_eval(blk, h, table)
        feat = h.reshape(h.shape[0], h.shape[3]) if h.shape[1] == 1 and h.shape[2] == 1 else F.avgpool(h)
        fc = self.fc
        w = bnn._shadow(fc, "weight", fc.weight)
        if fc.act == 0:
            head = F.linear_xent_eval(feat.contiguous(), w, fc.bias, target, acc, want_logits=want_logits)
            if head is not None:
                return head[1]
        logits = F.gemm(feat.contiguous(), w, bias=fc.bias, act=fc.act, out_dtype=torch.float32)
        F.softmax_xent(logits, target, want_grad=False, acc=acc, loss_scale=1.0)
        return logits if want_logits else None

    # ------------------------------------------------------------------
    def build_workspace(self, device) -> torch.Tensor:
        """One fp32 buffer holding the forward/backward statistic sums of every
        BatchNorm layer (4*C each), zeroed by ONE memset per training step."""
        bns = [m for m in self.modules() if isinstance(m, bnn.BatchNorm2d)]
        total = sum(4 * m.num_features for m in bns)
        ws = torch.zeros(total, dtype=torch.float32, device=device)
        off = 0
        for m in bns:
            m.workspace = ws[off: off + 4 * m.num_features]
            off += 4 * m.num_features
        self.stats_workspace = ws if bns else None      # a GroupNorm model has no batch statistics
        # convolution -> BatchNorm pairs: the conv GEMM's epilogue accumulates the batch statistics straight
        # into the BatchNorm's workspace, so the separate statistics pass over the activation disappears
        for parent in self.modules():
            for conv_name, bn_name in (("conv1", "bn1"), ("conv2", "bn2"), ("conv3", "bn3")):
                conv, bn = getattr(parent, conv_name, None), getattr(parent, bn_name, None)
                if isinstance(conv, bnn.Conv2d) and isinstance(bn, bnn.BatchNorm2d):
                    conv.bn_ws = bn.workspace
            if isinstance(parent, _Downsample) and isinstance(parent[1], bnn.BatchNorm2d):
                parent[0].bn_ws = parent[1].workspace
        return ws


def resnet18(num_classes: int = 10, **kw) -> ResNet:
    """``norm="group", groups=G``: GroupNorm(G, C) in place of every BatchNorm."""
    kw.setdefault("name", "resnet18" if kw.get("norm", "batch") == "batch" else "resnet18_gn")
    return ResNet(BasicBlock, [2, 2, 2, 2], num_classes=num_classes, **kw)


def resnet50(num_classes: int = 1000, **kw) -> ResNet:
    kw.setdefault("name", "resnet50" if kw.get("norm", "batch") == "batch" else "resnet50_gn")
    return ResNet(Bottleneck, [3, 4, 6, 3], num_classes=num_classes, **kw)
