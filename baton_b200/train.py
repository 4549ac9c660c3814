"""Local-SGD loop run by every federated client between two aggregations.

Parity target: demo ``Model.train`` (reference demo.py:29-49): one ``randperm``
per call (demo.py:33, kept as the default -- quirk 12), plain SGD, per epoch a
pass over ``torch.split(idxs, batch_size)`` with zero_grad / gather / forward /
loss / backward / step, returning one running-mean loss per epoch.

Two executions of the same contract:

* ``run_local_sgd`` -- portable PyTorch loop (CPU, gloo plumbing config, test
  oracle).  The loss is accumulated in a tensor and read once per epoch (the
  reference does ``float(loss)`` per batch, utils.py:88).
* ``GraphedLocalSGD`` (CUDA) -- the whole step (on-device batch gather, forward,
  loss, backward, fused arena SGD, loss accumulation) is captured once into a
  CUDA graph and replayed per batch; parameters, gradients and momentum live in
  the flat arena, so the optimizer takes at most one launch per step beyond the
  weight-gradient GEMM epilogues instead of one launch per tensor.  No host
  synchronisation inside an epoch.

Every trainer takes ``prox_mu`` (FedProx, Li et al. 2020): the step adds
``prox_mu * (w - w_global)`` to the gradient, ``w_global`` being the global model
the round started from.  ``prox_mu = 0`` is plain SGD.  The arena trainers also
take ``corr`` (SCAFFOLD, Karimireddy et al. 2020): an fp32 buffer indexed like
the parameters, holding ``c - c_i``, that every step adds to the gradient.

Every trainer also takes ``optimizer="adamw"`` (with ``betas`` and ``eps``): the local
steps are those of ``torch.optim.AdamW`` with one parameter group, created fresh for
each run -- the reference builds its optimizer inside every ``train()`` call.  The
step count ``t`` runs across the epochs of one run.  AdamW takes no momentum,
Nesterov, FedProx or SCAFFOLD term.

Every trainer also takes ``augment="crop" | "flip" | "crop_flip"`` with ``augment_padding`` (``data/augment.py``):
each epoch's batches are randomly cropped from the zero-padded image and flipped, fresh draws per sample and epoch.
``GraphedLocalSGD`` does it inside the epoch's batch gather (``F.gather_augment``); the CPU trainers call the host
reference per batch.  ``augment_seed`` / ``augment_stream`` pick the draws (``data/augment.py: AugmentStreams``).

Cross-entropy trainers also take ``mix="mixup" | "cutmix" | "mixup_cutmix"`` with ``mix_alpha``, and
``label_smoothing`` (``data/mix.py``): each batch is mixed with itself rolled by one under one lambda per batch, and
the loss is the soft-target cross-entropy.  ``GraphedLocalSGD`` mixes inside the same batch gather and applies the soft
target in the fused loss kernels; the CPU trainers call the host reference.  Mixing draws from the augmentation key
and stream, so it takes the same ``augment_seed`` / ``augment_stream``.

Every trainer also takes ``max_grad_norm`` (``C > 0``): ``torch.nn.utils.clip_grad_norm_(parameters, C)`` of every
step's gradient right after backward, before weight decay and the FedProx, SCAFFOLD, momentum or AdamW terms act.
``GraphedLocalSGD`` runs one norm kernel per step (``F.grad_norm_clip``) and the clipped optimizer kernels; the CPU
trainers call ``clip_grad_norm_``.  ``last_grad_norms()`` returns the pre-clip norms of the last run.
"""
from __future__ import annotations

import contextlib
import gc
from collections import OrderedDict
from typing import Callable, List, Optional, Tuple

import numpy as np
import torch
from torch import nn

from .data.augment import AugmentStreams, check_augment, check_shard, gather_augment_reference
from .data.mix import (MIX_ROW, check_mix, check_mix_loss, check_mix_shard, mix_batch_reference, mix_rows, mix_table,
                       soft_cross_entropy, soft_hits)
from .utils.progress import EpochProgress


def _loss_fn(kind):
    if callable(kind):
        return kind
    if kind == "mse":
        return nn.functional.mse_loss
    if kind in ("ce", "cross_entropy"):
        return nn.functional.cross_entropy
    raise ValueError("unknown loss {!r}".format(kind))


def check_prox_mu(prox_mu: float) -> float:
    """The FedProx coefficient as a float; ``ValueError`` unless it is a finite number >= 0."""
    mu = float(prox_mu)
    if not (0.0 <= mu < float("inf")):
        raise ValueError("prox_mu must be a finite number >= 0, got {!r}".format(prox_mu))
    return mu


def check_max_grad_norm(max_grad_norm: float) -> float:
    """The gradient-norm clip threshold as a float; ``ValueError`` unless it is a finite number >= 0 (0: no clipping)."""
    try:
        c = float(max_grad_norm)
    except (TypeError, ValueError):
        raise ValueError("max_grad_norm must be a finite number >= 0, got {!r}".format(max_grad_norm)) from None
    if not (0.0 <= c < float("inf")):
        raise ValueError("max_grad_norm must be a finite number >= 0, got {!r}".format(max_grad_norm))
    return c


def clip_coefficient(norm, max_grad_norm: float) -> np.ndarray:
    """The coefficient ``clip_grad_norm_`` multiplies the gradients by, as the device kernel computes it from its fp32
    norm: ``min(fl32(fl32(1 / fl32(norm + 1e-6)) * C), 1)`` with ``C`` rounded to fp32 and every operation rounded to
    fp32.  That is torch's ``clamp(reciprocal(norm + 1e-6) * C, max=1)`` bit for bit; a NaN norm gives NaN, an
    infinite one 0."""
    n = np.asarray(norm, dtype=np.float32)
    with np.errstate(divide="ignore", over="ignore", invalid="ignore"):
        c = (np.float32(1.0) / (n + np.float32(1e-6))) * np.float32(max_grad_norm)
    return np.where(c > np.float32(1.0), np.float32(1.0), c).astype(np.float32)


def _clip_grads(params, max_grad_norm: float):
    """``clip_grad_norm_`` of the step's gradients (2-norm, non-finite norms allowed); returns the pre-clip norm."""
    return nn.utils.clip_grad_norm_(params, max_grad_norm, error_if_nonfinite=False).detach()


def check_adamw(betas, eps) -> Tuple[Tuple[float, float], float]:
    """AdamW's ``(betas, eps)`` as floats; ``ValueError`` unless both betas are in [0, 1) and ``eps > 0`` (finite)."""
    try:
        b1, b2 = (float(b) for b in betas)
    except (TypeError, ValueError):
        raise ValueError("betas must be a pair of numbers, got {!r}".format(betas)) from None
    for name, b in (("beta1", b1), ("beta2", b2)):
        if not 0.0 <= b < 1.0:
            raise ValueError("AdamW {} must be in [0, 1), got {!r}".format(name, b))
    eps = float(eps)
    if not 0.0 < eps < float("inf"):
        raise ValueError("AdamW eps must be a finite number > 0, got {!r}".format(eps))
    return (b1, b2), eps


def check_optimizer(optimizer: str, momentum: float = 0.0, nesterov: bool = False, prox_mu: float = 0.0,
                    corr=None) -> bool:
    """True for ``"adamw"``, False for ``"sgd"``; ``ValueError`` for another name, or for a local step that cannot
    combine its terms (``parallel/features.py``: AdamW with momentum, Nesterov, FedProx or SCAFFOLD, and SCAFFOLD's
    correction ``corr`` with FedProx)."""
    from .parallel.features import check_features
    check_features(optimizer=optimizer, momentum=momentum, nesterov=nesterov, prox_mu=prox_mu,
                   scaffold=corr is not None)
    return optimizer == "adamw"


def _add_prox_term(params, anchors, prox_mu: float) -> None:
    """FedProx: ``grad += prox_mu * (w - anchor)`` before the optimizer step (what the reference implementation does)."""
    with torch.no_grad():
        for p, a in zip(params, anchors):
            if p.grad is not None:
                p.grad.add_(p.detach() - a, alpha=prox_mu)


def _check_corr(corr, arena) -> None:
    if corr is not None and (corr.dtype != torch.float32 or not corr.is_contiguous() or corr.numel() < arena.n_param):
        raise ValueError("corr must be a contiguous fp32 buffer covering the arena's parameters")


def run_local_sgd(model: nn.Module, X: torch.Tensor, y: torch.Tensor, *, n_epoch: int = 32,
                  lr: float = 0.001, batch_size: int = 32, momentum: float = 0.0,
                  weight_decay: float = 0.0, loss: "str | Callable" = "mse",
                  verbose: bool = False, reshuffle_each_epoch: bool = False,
                  generator: Optional[torch.Generator] = None, prox_mu: float = 0.0, optimizer: str = "sgd",
                  betas: Tuple[float, float] = (0.9, 0.999), eps: float = 1e-8, augment: Optional[str] = None,
                  augment_padding: int = 4, augment_seed: Optional[int] = None,
                  augment_stream: Optional[int] = None, mix: Optional[str] = None, mix_alpha: float = 1.0,
                  label_smoothing: float = 0.0, max_grad_norm: float = 0.0) -> List[float]:
    """Portable local SGD; returns the per-epoch mean loss.  ``prox_mu > 0``: FedProx, anchored on the parameters as
    they are on entry -- the global model the worker has just loaded.  ``optimizer="adamw"``: a fresh
    ``torch.optim.AdamW(lr, betas, eps, weight_decay)`` instead of SGD.  ``augment``: random crop / flip of every
    batch; the model keeps the key and run counter (``AugmentStreams``) across calls.  ``mix`` / ``label_smoothing``:
    mixup / CutMix of every batch and the soft-target loss (``data/mix.py``).  ``max_grad_norm > 0``:
    ``clip_grad_norm_(parameters, max_grad_norm)`` right after every backward, before the FedProx term."""
    criterion = _loss_fn(loss)
    prox_mu = check_prox_mu(prox_mu)
    max_grad_norm = check_max_grad_norm(max_grad_norm)
    adam = check_optimizer(optimizer, momentum, prox_mu=prox_mu)
    mixc = _mix_setup(mix, mix_alpha, label_smoothing, loss)
    streams = model.__dict__.setdefault("_augment_streams", AugmentStreams())
    aug = _augment_setup(streams, X, augment, augment_padding, augment_seed, augment_stream, mixc)
    drop = _dropout_setup(model, streams, aug, augment_seed, augment_stream)
    n = X.shape[0]
    if drop is not None:
        drop[0].begin(drop[1], drop[2], -(-n // batch_size), n_epoch, model.n_dropout_sites)
    try:
        return _run_local_sgd(model, X, y, n_epoch, lr, batch_size, momentum, weight_decay, verbose,
                              reshuffle_each_epoch, generator, prox_mu, adam, betas, eps, mixc, aug, max_grad_norm,
                              criterion, drop)
    finally:
        if drop is not None:
            drop[0].end()


def _run_local_sgd(model, X, y, n_epoch, lr, batch_size, momentum, weight_decay, verbose, reshuffle_each_epoch,
                   generator, prox_mu, adam, betas, eps, mixc, aug, max_grad_norm, criterion, drop):
    n = X.shape[0]
    nn.Module.train(model, True)
    params = list(model.parameters())
    anchors = [p.detach().clone() for p in params] if prox_mu > 0 else None
    if adam:
        betas, eps = check_adamw(betas, eps)
        optimizer = torch.optim.AdamW(params, lr=lr, betas=betas, eps=eps, weight_decay=weight_decay)
    else:
        optimizer = torch.optim.SGD(params, lr=lr, momentum=momentum,
                                    weight_decay=weight_decay)
    idxs = torch.randperm(n, generator=generator).to(X.device)
    loss_history: List[float] = []
    for epoch in range(n_epoch):
        if reshuffle_each_epoch and epoch > 0:
            idxs = torch.randperm(n, generator=generator).to(X.device)
        batches = torch.split(idxs, batch_size)
        rows = _host_mix_rows(mixc, aug, X, epoch, len(batches))
        batch_iter = EpochProgress(epoch, batches, verbose=verbose)
        for b, batch_idxs in enumerate(batch_iter):
            optimizer.zero_grad(set_to_none=True)
            if drop is not None:
                drop[0].at(epoch, b)
            xb = _host_batch(X, batch_idxs, aug, epoch, b * batch_size)
            target = y[batch_idxs]
            if mixc is not None:
                xb, soft = mix_batch_reference(xb, target, rows[b] if rows is not None else None, mixc.smoothing)
            output = model(xb)
            if output.shape != target.shape and target.dtype.is_floating_point:
                target = target.reshape(output.shape)  # (N,) vs (N,1) -- quirk 13
            loss_batch = criterion(output, target) if mixc is None else soft_cross_entropy(output, soft)
            batch_iter.update_loss(loss_batch)
            loss_batch.backward()
            if max_grad_norm > 0:
                _clip_grads(params, max_grad_norm)
            if anchors is not None:
                _add_prox_term(params, anchors, prox_mu)
            optimizer.step()
        loss_history.append(batch_iter.loss)
    return loss_history


def _augment_setup(streams: AugmentStreams, X, augment, augment_padding, augment_seed, augment_stream, mix=None):
    """``(config, key, stream)`` of a run, or None when it neither augments nor mixes (``config`` is None when it only
    mixes: mixing draws from the same key and stream); ``ValueError`` for a bad config or shard."""
    cfg = check_augment(augment, augment_padding)
    mixing = mix is not None and mix.kind is not None
    if cfg is None and not mixing:
        return None
    if cfg is not None:
        check_shard(cfg, X)
    check_mix_shard(mix, X)
    return (cfg,) + streams.next(augment_seed, augment_stream)


def _dropout_setup(model, streams: AugmentStreams, aug, augment_seed, augment_stream):
    """``(run, key, stream)`` of a run of a model with a nonzero dropout probability (``data/dropout.py``), or None.
    Dropout draws from the augmentation key and stream: those of ``aug`` when the run augments or mixes, else the
    next of ``streams``."""
    run = getattr(model, "dropout_run", None)
    if run is None or not getattr(model, "has_dropout", False):
        return None
    key, stream = aug[1:] if aug is not None else streams.next(augment_seed, augment_stream)
    return run, key, stream


def _mix_setup(mix, mix_alpha, label_smoothing, loss):
    """The run's :class:`~baton_b200.data.mix.MixConfig` (None: hard targets); ``ValueError`` for a bad config or a
    loss that is not the cross-entropy."""
    cfg = check_mix(mix, mix_alpha, label_smoothing)
    check_mix_loss(cfg, loss)
    return cfg


def _host_mix_rows(mixc, aug, X, epoch: int, n_batches: int):
    """The epoch's mix rows (``data/mix.py: mix_table``), or None when the run does not mix."""
    if mixc is None or mixc.kind is None:
        return None
    _, key, stream = aug
    return mix_table(key, stream, epoch, n_batches, mixc, X.shape[1], X.shape[2])


def _host_batch(X, idx, aug, epoch: int, s0: int):
    """``X[idx]``, augmented (host reference) for epoch positions ``s0 ..`` when ``aug`` crops or flips."""
    if aug is None or aug[0] is None:
        return X[idx]
    cfg, key, stream = aug
    return gather_augment_reference(X, idx, key, stream, epoch, cfg.padding, cfg.crop, cfg.flip, s0=s0)


def bn_fold_table(model: nn.Module, arena):
    """``(table, n_floats)``: the descriptor table of ``F.bn_fold_eval`` for every BatchNorm of an arena-adopted model
    (int64 ``[n_bn, 7]`` on the arena's device) and the size of its output, or ``None`` when the model has none.
    Sets each BatchNorm's ``eval_off``: where its eval scale (``C`` floats) and shift (the next ``C``) land in the
    output buffer, 8-float aligned."""
    import struct
    from .ops import nn as bnn
    rows, off = [], 0
    for name, m in model.named_modules():
        if not isinstance(m, bnn.BatchNorm2d):
            continue
        pre = name + "." if name else ""
        slot = lambda leaf: arena.slots[pre + leaf].offset if (pre + leaf) in arena.slots else -1   # noqa: E731
        eps_bits = struct.unpack("<i", struct.pack("<f", float(m.eps)))[0]
        rows.append([slot("weight"), slot("bias"), slot("running_mean"), slot("running_var"), off, m.num_features,
                     eps_bits])
        m.eval_off = off
        off += (2 * m.num_features + 7) // 8 * 8
    if not rows:
        return None
    return torch.tensor(rows, dtype=torch.int64).to(arena.device), off


def _eval_batch_generic(model, xb, yb, acc, loss_kind, F):
    """``model.eval()`` forward of one batch, then the summed loss (and #correct for classification) into ``acc``."""
    with torch.no_grad():
        out = model(xb)
    if loss_kind in ("ce", "cross_entropy"):
        out2 = out.reshape(-1, out.shape[-1])
        F.softmax_xent(out2 if out2.stride(-1) == 1 else out2.contiguous(), yb, want_grad=False, acc=acc,
                       loss_scale=1.0)
    else:
        # per-sample mean squared error, summed over the batch: the mean over samples is mse_loss of the whole shard
        per_row = max(1, out.numel() // max(1, out.shape[0]))
        F.load().mse(out.contiguous(), yb.reshape(out.shape).contiguous().float(), None, acc, 1.0 / per_row)


@contextlib.contextmanager
def _no_gc_during_capture():
    """Keep the cyclic garbage collector from running while a CUDA graph is captured.  A model and its graphed trainer
    reference each other, so a dropped engine's graphs are freed only by the collector, which can run at any allocation.
    Destroying a graph is not permitted while a stream is capturing, and the attempt invalidates the capture in progress;
    deferred until after the capture, it is harmless."""
    enabled = gc.isenabled()
    gc.disable()
    try:
        yield
    finally:
        if enabled:
            gc.enable()


class GraphedLocalSGD:
    """CUDA local-SGD engine for an arena-adopted model.

    One *epoch* -- ``n // batch_size`` steps of {on-device batch gather, forward,
    fused loss, hand-written backward, SGD, loss accumulation} -- is captured into
    a single CUDA graph and replayed once per epoch, so the host issues one launch
    per epoch and never synchronises inside a round: the per-epoch losses are read
    back together when the round ends.

    A model that offers ``explicit_step`` trains with it whenever it runs in bf16
    with the cross-entropy loss; MXFP8, MSE and models without one go through
    autograd.  ``run(prox_mu > 0)`` adds FedProx's pull toward ``arena.global_w`` in every
    SGD kernel.  SGD runs in one of two places.  In a hand-scheduled step the
    split-K = 1 convolution weight-gradient GEMMs apply it in their epilogue and
    ``fused_sgd_segments`` updates the rest of the arena.  The epoch's last step
    (it also writes the upload copy), ragged eager steps and autograd steps run
    ONE ``fused_sgd`` kernel over the whole arena instead.

    ``run(optimizer="adamw")`` runs AdamW in the same three places.  Its first moment is
    ``arena.momentum`` and its second ``arena.adam_v``.  The per-step bias corrections
    come from a table of rows (``F.adamw_rows``), one row per local step of the run.  It
    is built on the host when the run starts and copied to the device once.  Before each
    epoch's replay, that epoch's rows are copied into the epoch graph's row buffer, and
    captured step ``s`` reads row ``s``.  The ragged eager step uses the buffer's last row.

    ``run(augment=...)`` gathers the batches through ``F.gather_augment`` instead of ``F.gather_rows``.  Its per-epoch
    words ``{epoch, stream_lo, stream_hi}`` follow the AdamW rows: one ``[n_epoch, 3]`` device table per run (written
    on the device, see ``_aug_words``), and before each replay that epoch's row is copied into the graph's word
    buffer.  The key is a launch argument, so
    it is part of the epoch graph's key.

    ``run(mix=...)`` gathers through the mixing form of the same kernel (``F.gather_augment(mix_rows=...)``) and
    trains on the soft-target loss kernels (``label_smoothing`` alone needs only those).  The run's mix rows
    (``data/mix.py: mix_rows``, ``[n_epoch, steps, 8]``) are built on the host in pinned memory and copied without a
    host synchronisation; before each replay that epoch's rows are copied into the graph's ``[steps, 8]`` row buffer,
    which the gather reads whole and captured step ``s`` passes row ``s`` of to the loss.  Whether the run mixes and
    its smoothing (a launch argument) are part of the graph key; lambda and the boxes are not.

    ``model`` must already be adopted by a :class:`~baton_b200.parallel.arena.ParamArena`
    (``arena``); the engine is what ``FederatedModule.local_train`` dispatches to
    for CUDA shards (``model._graphed_trainer``).
    """

    EVAL_GRAPHS_MAX = 4      # captured evaluation passes kept (each holds its activations in a private pool)

    def __init__(self, model: nn.Module, arena, *, loss: str = "ce", nesterov: bool = False,
                 use_graph: bool = True, input_dtype=torch.bfloat16):
        from .ops import functional as F
        from .ops import nn as bnn
        self.F, self.bnn = F, bnn
        self.model, self.arena = model, arena
        self.loss_kind = loss
        self.nesterov = nesterov
        self.use_graph = use_graph
        self.input_dtype = input_dtype
        self._seg_tables = {}
        self.k3_join = None           # set by the engine: callable joining the round-end collective (enables the graph split)
        self._first_gemm_hook = None
        self.pack = None              # set by the engine: FedAvgSession.pack_spec() -> last SGD step emits the upload copy
        self.emitted_wire = False
        self.graph_emits_wire = False
        dev = arena.device
        self.device = dev
        # [lr, momentum, wd, dampening, prox_mu, clip coefficient]; the last is written on the device by a clipped step
        self.hyper = torch.zeros(6, dtype=torch.float32, device=dev)
        self.prox = False             # FedProx: every SGD kernel of the step reads the anchor arena.global_w
        self.corr = None              # SCAFFOLD: every SGD kernel of the step reads this correction c - c_i
        self.adam = False             # AdamW: every optimizer kernel of the step reads its step row and arena.adam_v
        self._adam_table = (None, None)   # (host key, device [n_epoch * steps, ADAMW_ROW] rows of the run)
        self._aug = None              # augmentation of the current run: (AugmentConfig, key, stream) or None
        self._aug_streams = AugmentStreams()
        self._aug_table = None        # device [epochs, 3] per-epoch words of augmenting runs (see _aug_words)
        self._mix = None              # MixConfig of the current run (mixing and / or label smoothing) or None
        self._drop = None             # dropout of the current run: (DropoutRun, key, stream) or None
        self.clip = False             # gradient-norm clipping: each step runs the norm kernel, then a clipped optimizer
        self.max_norm = torch.zeros(1, dtype=torch.float32, device=dev)   # its threshold, read by the norm kernel
        self._max_norm_host = None
        self._norm_work = None        # the norm kernel's partials and arrival counter
        self.grad_norms = None        # device [n_epoch, steps] pre-clip norms of the last run (None: no clipping)
        self.loss_acc = torch.zeros(2, dtype=torch.float32, device=dev)
        self._graphs = {}           # (n, batch, x_shape, y_shape) -> captured epoch
        self._hyper_host = None
        self.n_kernels_per_step = None
        self.last_stats = {}
        self.eval_acc = torch.zeros(2, dtype=torch.float32, device=dev)   # evaluation only: [loss sum, #correct]
        self._eval_graphs = OrderedDict()    # captured evaluation passes, least recently used first
        self._fold = None
        self.eval_launches = None     # Counter of the kernels in the last captured evaluation pass

    # -------------------------------------------------------------- one SGD step (capturable)
    def _loss(self, out, yb, mix=None):
        if self.loss_kind in ("ce", "cross_entropy"):
            loss, stats = self.bnn.cross_entropy(out, yb) if mix is None else self.bnn.cross_entropy(out, yb, mix=mix)
            return loss, stats
        loss = self.bnn.mse_loss(out, yb)
        return loss, torch.stack([loss.detach(), torch.zeros_like(loss.detach())])

    def _gather(self, X, y, idx, s0=0, words=None, mix_rows=None, bsz=None):
        """``X[idx], y[idx]``; with augmentation or mixing on, ``X`` is gathered by ``F.gather_augment`` for epoch
        positions ``s0 ..`` with the device words ``words`` (and the epoch's mix rows ``mix_rows``, batches of
        ``bsz``)."""
        F = self.F
        if self._aug is not None:
            cfg, key, _ = self._aug
            pad, crop, flip = (cfg.padding, cfg.crop, cfg.flip) if cfg is not None else (0, False, False)
            xb = F.gather_augment(X, idx, words, key, pad, crop=crop, flip=flip, s0=s0, mix_rows=mix_rows, batch=bsz)
        else:
            xb = F.gather_rows(X, idx)
        yb = F.gather_rows(y, idx) if y.dtype == torch.int64 and y.dim() == 1 else y.index_select(0, idx)
        return xb, yb

    def _step(self, X, y, idx, batch=None, emit_wire=False, fuse_sgd=True, row=None, s0=0, words=None, mix_rows=None,
              bsz=None, norm=None):
        """One SGD step on ``X[idx], y[idx]`` (or on the already gathered ``batch``).  ``emit_wire``: last step of
        an epoch -- the optimizer kernel also writes the upload copy for the round-end collective (``self.pack``).
        ``fuse_sgd=False``: no optimizer epilogue in the weight-gradient GEMMs (one optimizer pass over the arena).
        ``row``: with AdamW, the device row of this step's coefficients (``F.adamw_rows``).  ``s0``, ``words``: the
        epoch position of ``idx[0]`` and the device words of an augmenting gather.  ``mix_rows``, ``bsz``: the
        epoch's device mix rows and the batch size of a mixing run; the loss reads row ``s0 // bsz``.  ``norm``: with
        clipping on, the device scalar this step writes its pre-clip gradient norm to."""
        F = self.F
        xb, yb = batch if batch is not None else self._gather(X, y, idx, s0, words, mix_rows, bsz)
        if self._drop is not None:
            self._drop[0].at(0, s0 // bsz, words)       # the kernels read the epoch from `words`
        mix = None
        if self._mix is not None:
            mix = (mix_rows[s0 // bsz] if mix_rows is not None else None, self._mix.smoothing)
        soft = {"mix": mix} if mix is not None else {}
        ws = getattr(self.model, "stats_workspace", None)
        if ws is not None and not getattr(self.model, "zeroes_own_workspace", False):
            ws.zero_()
        explicit = getattr(self.model, "explicit_step", None)
        if getattr(self.model, "compute_dtype", "bf16") != "bf16":
            explicit = None            # the hand-scheduled step drives the bf16 conv kernels; MXFP8 convs go through autograd
        a = self.arena
        bf = a.theta_bf16
        anchor = a.global_w if self.prox else None
        hyper = row if self.adam else self.hyper
        adam_v = a.adam_v if self.adam else None
        if explicit is not None and self.loss_kind in ("ce", "cross_entropy"):
            # hand-scheduled forward + loss + backward (no autograd engine): two-piece block gradients, parallel shortcut
            # branch; the loss kernel accumulates straight into the epoch's running sums
            if fuse_sgd and not emit_wire:
                # the split-K = 1 convolution weight gradients apply SGD in their GEMM epilogue; one launch covers the rest.
                # A clipped step cannot: its coefficient needs the last gradient.  Its GEMMs only record the no-gradient
                # taps, which the leftover pass (then over the whole arena) still skips.
                with self.bnn.SGD_EPI.open(a, hyper, self.nesterov, prox=self.prox, corr=self.corr,
                                           adam_v=adam_v, fuse=not self.clip) as epi:
                    explicit(xb, yb, loss_acc=self.loss_acc, after_first_gemm=self._first_gemm_hook, **soft)
                if self.clip:
                    self._grad_norm(norm, hyper)
                F.fused_sgd_segments(a.theta, a.grad, hyper, self._segment_table(epi.fused, epi.nograd),
                                     a.momentum, bf, nesterov=self.nesterov, prox_anchor=anchor, corr=self.corr,
                                     adam_v=adam_v, clip=self.clip)
                self.emitted_wire = False
                return
            explicit(xb, yb, loss_acc=self.loss_acc, after_first_gemm=self._first_gemm_hook, **soft)
            stats = None
        else:
            out = self.model(xb)
            loss, stats = self._loss(out, yb, mix)
            loss.backward()
            self.bnn.WGRAD.join()      # weight-gradient GEMMs run on a side stream; they must land before the step
        # one optimizer pass over the whole arena; the epoch's last step also emits the upload copy
        pack = self.pack if emit_wire else None
        if self.clip:
            self._grad_norm(norm, hyper)
        F.fused_sgd(a.theta[: a.n_param], a.grad, hyper, a.momentum,
                    bf[: a.n_param] if bf is not None else None, zero_grad=True, nesterov=self.nesterov, pack=pack,
                    prox_anchor=anchor[: a.n_param] if anchor is not None else None,
                    corr=self.corr[: a.n_param] if self.corr is not None else None, adam_v=adam_v, clip=self.clip)
        self.emitted_wire = pack is not None
        if stats is not None:
            self.loss_acc.add_(stats)

    def _grad_norm(self, norm, hyper):
        """The norm kernel of a clipped step: ``||grad[0:n_param]||`` into ``norm`` and the clip coefficient into the
        slot of ``hyper`` (the SGD hyper-parameters or the step's AdamW row) the clipped optimizer kernels read."""
        F = self.F
        slot = F.ADAMW_ROW_CLIP if self.adam else F.SGD_HYPER_CLIP
        F.grad_norm_clip(self.arena.grad[: self.arena.n_param], self.max_norm, self._norm_work, norm,
                         hyper[slot: slot + 1])

    def _segment_table(self, fused, nograd):
        """Device chunk table of the leftover optimizer pass, built once per set of epilogue-updated ranges (they only
        change with the batch shape, so every step of a captured epoch reuses the table its warm-up built)."""
        key = (tuple(fused), tuple(nograd))
        table = self._seg_tables.get(key)
        if table is None:
            segs = self.F.sgd_segments(self.arena.n_param, fused, nograd)
            table = self._seg_tables[key] = torch.tensor(segs, dtype=torch.int64).view(-1, 3).to(self.device)
        return table

    def _set_hyper(self, lr, momentum, weight_decay, dampening=0.0, prox_mu=0.0):
        vals = (float(lr), float(momentum), float(weight_decay), float(dampening), float(prox_mu))
        if vals != self._hyper_host:
            self.hyper[:5].copy_(torch.tensor(vals, dtype=torch.float32))
            self._hyper_host = vals

    def _set_max_norm(self, max_grad_norm: float):
        if max_grad_norm != self._max_norm_host:
            self.max_norm.fill_(max_grad_norm)
            self._max_norm_host = max_grad_norm
        if self._norm_work is None:
            self._norm_work = torch.zeros(self.F.load().GRAD_NORM_WORK_WORDS, dtype=torch.int64, device=self.device)

    def _adam_rows(self, lr, betas, eps, weight_decay, n_epoch, steps):
        """Device ``[n_epoch * steps, ADAMW_ROW]`` AdamW coefficients of every local step of a run (step ``t`` counts
        across epochs); copied to the device only when they change."""
        key = (float(lr), tuple(betas), float(eps), float(weight_decay), n_epoch, steps)
        if self._adam_table[0] != key:
            rows = self.F.adamw_rows(lr, betas, eps, weight_decay, 1, n_epoch * steps)
            self._adam_table = (key, rows.to(self.device))
        return self._adam_table[1]

    def _aug_words(self, stream: int, n_epoch: int):
        """Device int32 ``[n_epoch, 3]`` per-epoch words ``{epoch, stream_lo, stream_hi}`` of an augmenting run.  The
        table persists; a run rewrites the stream columns with two fills, so no host copy (and no host
        synchronisation) is needed."""
        t = self._aug_table
        if t is None or t.shape[0] < n_epoch:
            t = self._aug_table = torch.zeros(n_epoch, 3, dtype=torch.int32, device=self.device)
            t[:, 0].copy_(torch.arange(n_epoch, dtype=torch.int32, device=self.device))
        for col, word in ((1, stream & 0xFFFFFFFF), (2, (stream >> 32) & 0xFFFFFFFF)):
            t[:, col].fill_(word - (1 << 32) if word >> 31 else word)
        return t[:n_epoch]

    def _mix_rows(self, n_epoch: int, steps: int, X):
        """Device int32 ``[n_epoch, steps, 8]`` mix rows of a mixing run: built on the host in pinned memory and copied
        asynchronously (no host synchronisation)."""
        _, key, stream = self._aug
        host = mix_rows(key, stream, n_epoch, steps, self._mix, X.shape[1], X.shape[2]).pin_memory()
        return host.to(self.device, non_blocking=True)

    # -------------------------------------------------------------- epoch graph
    def _capture(self, X, y, n_steps, batch_size, rows=None, steps=None):
        """``rows``: with AdamW, the device row buffer captured step ``s`` reads row ``s`` of (holding the first
        epoch's rows, which the warm-up steps use too); kept in the returned entry.  With augmentation on, the
        gather reads the entry's word buffer ``words``; with mixing on, the entry's ``[steps, 8]`` mix rows ``mix``.
        With clipping on, captured step ``s`` writes its gradient norm to ``norms[s]`` of the entry."""
        perm = torch.zeros(n_steps * batch_size, dtype=torch.int64, device=self.device)
        words = (torch.zeros(3, dtype=torch.int32, device=self.device)
                 if self._aug is not None or self._drop is not None else None)
        mixbuf = (torch.zeros(steps, MIX_ROW, dtype=torch.int32, device=self.device)
                  if self._mix is not None and self._mix.kind is not None else None)
        norms = torch.zeros(steps, dtype=torch.float32, device=self.device) if self.clip else None
        perm.copy_(torch.arange(n_steps * batch_size, device=self.device) % X.shape[0])
        side = torch.cuda.Stream(device=self.device)
        side.wait_stream(torch.cuda.current_stream(self.device))
        with torch.cuda.stream(side):   # warm-up outside capture (allocator, lazy init, autograd)
            # hyper lr=0 during warm-up/capture would still move BN statistics; save/restore the state
            snap = self.arena.theta.clone()
            snap_i = self.arena.int_arena.clone()
            snap_m = self.arena.momentum.clone() if self.arena.momentum is not None else None
            for _ in range(2):
                self._step(X, y, perm[:batch_size], row=rows[0] if rows is not None else None, words=words,
                           mix_rows=mixbuf, bsz=batch_size, norm=norms[0:1] if norms is not None else None)
        torch.cuda.current_stream(self.device).wait_stream(side)
        torch.cuda.synchronize(self.device)
        from .ops._ext import total_launches
        graph = torch.cuda.CUDAGraph()
        graph2 = None
        c0 = total_launches()

        def body():
            # the epoch's batches are gathered by ONE launch pair (a permuted copy of the shard, 25 MB for the
            # flagship config) instead of two latency-bound gathers at the head of every step
            Xp, yp = self._gather(X, y, perm, 0, words, mixbuf, batch_size)
            for s in range(n_steps):
                self._step(X, y, None, batch=(Xp[s * batch_size:(s + 1) * batch_size],
                                              yp[s * batch_size:(s + 1) * batch_size]),
                           emit_wire=(s == n_steps - 1 and self.pack is not None),
                           row=rows[s] if rows is not None else None, s0=s * batch_size, words=words, mix_rows=mixbuf,
                           bsz=batch_size, norm=norms[s:s + 1] if norms is not None else None)
            self.graph_emits_wire = self.pack is not None

        if (self.k3_join is not None and hasattr(self.model, "explicit_step")
                and getattr(self.model, "compute_dtype", "bf16") == "bf16"):
            # bcast_gemm (K3): the epoch is captured as TWO graphs that share one memory pool.  Graph 1 ends right after
            # the first convolution's GEMM of the first step -- everything in it either does not touch the parameter
            # arena (batch gather, im2col) or acquires the collective's arrival flags (weight staging, TMA producer of
            # the GEMM), so it is replayed WITHOUT waiting for the round-end collective that is still running on its
            # side stream.  Graph 2 (the rest of the epoch) is replayed after the join.
            graph2 = torch.cuda.CUDAGraph()
            pool = torch.cuda.graph_pool_handle()
            cap = torch.cuda.Stream(device=self.device)
            cap.wait_stream(torch.cuda.current_stream(self.device))
            state = {"cut": False}

            def cut():
                if not state["cut"]:
                    state["cut"] = True
                    graph.capture_end()
                    graph2.capture_begin(pool=pool)
            self._first_gemm_hook = cut
            with torch.cuda.stream(cap), _no_gc_during_capture():
                graph.capture_begin(pool=pool)
                try:
                    body()
                finally:
                    self._first_gemm_hook = None
                (graph2 if state["cut"] else graph).capture_end()
            torch.cuda.current_stream(self.device).wait_stream(cap)
            if not state["cut"]:
                graph2 = None
        else:
            with _no_gc_during_capture(), torch.cuda.graph(graph):
                body()
        self.kernels_per_epoch = total_launches() - c0      # our kernels inside one epoch graph
        self.n_kernels_per_step = self.kernels_per_epoch // max(1, n_steps)
        # undo the side effects of warm-up + capture-time execution (capture does not execute,
        # warm-up did)
        self.arena.theta.copy_(snap)
        self.arena.int_arena.copy_(snap_i)
        if snap_m is not None:
            self.arena.momentum.copy_(snap_m)
        self.arena.grad.zero_()
        self.arena.sync_shadow()
        self.loss_acc.zero_()
        return {"graph": graph, "graph2": graph2, "perm": perm, "X": X, "y": y, "rows": rows, "words": words,
                "mix": mixbuf, "norms": norms}

    # -------------------------------------------------------------- evaluation
    def _eval_pass(self, X, y, batch_size, explicit):
        """One pass over ``X, y``: the BatchNorm fold at its head (the running statistics of this round), every full
        batch and the ragged last one.  Capturable; writes only ``eval_acc`` and the fold table."""
        self.eval_acc.zero_()
        if explicit:
            self._eval_head()
        n = X.shape[0]
        for s in range(0, n, batch_size):
            xb, yb = X[s: s + batch_size], y[s: s + batch_size]
            if explicit:
                self.model.explicit_eval(xb, yb, self.eval_acc)
            else:
                _eval_batch_generic(self.model, xb, yb, self.eval_acc, self.loss_kind, self.F)

    def _eval_head(self):
        """What an ``explicit_eval`` pass reads and the arena determines: the BatchNorm fold, the pass's weights."""
        table, out = self._fold
        self.F.bn_fold_eval(self.arena.theta, table, out)
        self.model.prepare_eval()

    def evaluate(self, X, y, batch_size: int = 512):
        """Loss and accuracy of the model as it stands (in eval mode) on a device-resident shard, without touching the
        arena, the training accumulators or the BatchNorm state.  Returns ``(loss_sum, correct, n)`` as floats: the
        summed per-sample loss (cross-entropy, or the per-sample mean squared error) and the number of correct
        predictions (0 for regression).  The whole pass is captured into ONE CUDA graph per shard (shape and
        address); a replay re-folds the BatchNorms from the current running statistics."""
        assert X.is_cuda, "GraphedLocalSGD.evaluate needs a device-resident shard"
        n = X.shape[0]
        if n == 0:
            return 0.0, 0.0, 0.0
        batch_size = max(1, min(batch_size, n))
        explicit = (hasattr(self.model, "explicit_eval") and hasattr(self.model, "prepare_eval")
                    and getattr(self.model, "compute_dtype", "bf16") == "bf16" and self.loss_kind in ("ce", "cross_entropy"))
        if explicit and self._fold is None:
            fold = bn_fold_table(self.model, self.arena)
            if fold is None:
                self._fold = False        # no BatchNorm to fold (a GroupNorm ResNet): the generic eval forward, every call
            else:
                table, size = fold
                out = torch.zeros(size, dtype=torch.float32, device=self.device)
                self._fold = (table, out)
                self.model.eval_bn_table = out
        if self._fold is False:
            explicit = False
        was_training = self.model.training
        nn.Module.train(self.model, False)
        try:
            if self.use_graph:
                key = (n, batch_size, tuple(X.shape[1:]), tuple(y.shape[1:]), X.dtype, y.dtype, X.data_ptr(),
                       y.data_ptr(), explicit)
                graph = self._eval_graphs.get(key)
                if graph is None:
                    while len(self._eval_graphs) >= self.EVAL_GRAPHS_MAX:
                        self._eval_graphs.popitem(last=False)       # frees that graph and its memory pool
                    graph = self._eval_graphs[key] = self._capture_eval(X, y, batch_size, explicit)
                self._eval_graphs.move_to_end(key)
                graph.replay()
            else:
                self._eval_pass(X, y, batch_size, explicit)
            loss_sum, correct = self.eval_acc.tolist()
        finally:
            nn.Module.train(self.model, was_training)
        return float(loss_sum), float(correct), float(n)

    def _capture_eval(self, X, y, batch_size, explicit):
        from .ops._ext import launch_counts
        cur = torch.cuda.current_stream(self.device)
        side = torch.cuda.Stream(device=self.device)
        side.wait_stream(cur)
        with torch.cuda.stream(side):   # warm-up outside capture (lazy init, kernel attributes); no state is written
            self._eval_pass(X, y, batch_size, explicit)
        cur.wait_stream(side)
        torch.cuda.synchronize(self.device)
        graph = torch.cuda.CUDAGraph()
        c0 = launch_counts()
        with _no_gc_during_capture(), torch.cuda.graph(graph):
            self._eval_pass(X, y, batch_size, explicit)
        self.eval_launches = launch_counts() - c0
        self.eval_captures = getattr(self, "eval_captures", 0) + 1
        return graph

    # -------------------------------------------------------------- public
    @torch.no_grad()
    def _shuffle_into(self, perm, n, generator=None):
        perm.copy_(torch.randperm(n, device=self.device)[: perm.numel()])

    def run(self, X, y, n_epoch: int = 1, lr: float = 0.001, batch_size: int = 32, momentum: float = 0.0,
            weight_decay: float = 0.0, reshuffle_each_epoch: bool = False, return_device: bool = False,
            prox_mu: float = 0.0, corr: Optional[torch.Tensor] = None, optimizer: str = "sgd",
            betas: Tuple[float, float] = (0.9, 0.999), eps: float = 1e-8, augment: Optional[str] = None,
            augment_padding: int = 4, augment_seed: Optional[int] = None, augment_stream: Optional[int] = None,
            mix: Optional[str] = None, mix_alpha: float = 1.0, label_smoothing: float = 0.0,
            max_grad_norm: float = 0.0, **_ignored):
        """``prox_mu > 0``: FedProx toward ``arena.global_w``, the global model the round started from.  ``corr``:
        SCAFFOLD's correction ``c - c_i`` (fp32 device buffer of ``arena.n_param`` elements), added to every step's
        gradient; it is read at replay, so the caller may rewrite it between runs.  ``optimizer="adamw"``: the steps of
        a fresh ``torch.optim.AdamW(lr, betas, eps, weight_decay)`` instead of SGD.  ``augment``: random crop / flip
        in the batch gather (``data/augment.py``); ``augment_seed`` (None: a random key per trainer) and
        ``augment_stream`` (None: this trainer's count of augmenting runs) pick the draws.  ``mix`` (with
        ``mix_alpha``) and ``label_smoothing``: mixup / CutMix in the same gather and the soft-target loss
        (``data/mix.py``), drawn from the same key and stream.  ``max_grad_norm > 0``: ``clip_grad_norm_`` of every
        step's gradient before the optimizer's terms are added (the norm kernel, then the clipped optimizer kernels);
        the threshold is read from device memory, so a new one replays the same graph."""
        assert X.is_cuda, "GraphedLocalSGD needs a device-resident shard"
        prox_mu = check_prox_mu(prox_mu)
        max_grad_norm = check_max_grad_norm(max_grad_norm)
        if prox_mu > 0 and self.arena.global_w is None:
            raise ValueError("prox_mu > 0 needs the arena's global copy (ParamArena(keep_global=True))")
        _check_corr(corr, self.arena)
        self.adam = check_optimizer(optimizer, momentum, self.nesterov, prox_mu, corr)
        if self.adam:
            betas, eps = check_adamw(betas, eps)
        self._mix = _mix_setup(mix, mix_alpha, label_smoothing, self.loss_kind)
        self._aug = _augment_setup(self._aug_streams, X, augment, augment_padding, augment_seed, augment_stream,
                                   self._mix)
        self._drop = _dropout_setup(self.model, self._aug_streams, self._aug, augment_seed, augment_stream)
        n = X.shape[0]
        batch_size = min(batch_size, n)
        n_steps = n // batch_size
        tail = n - n_steps * batch_size
        steps = n_steps + (1 if tail else 0)
        if self._drop is None:
            return self._run(X, y, n_epoch, lr, batch_size, momentum, weight_decay, reshuffle_each_epoch, return_device,
                             prox_mu, corr, betas, eps, max_grad_norm, n, n_steps, tail, steps)
        run, key, stream = self._drop
        run.begin(key, stream, steps, n_epoch, self.model.n_dropout_sites)
        try:
            return self._run(X, y, n_epoch, lr, batch_size, momentum, weight_decay, reshuffle_each_epoch, return_device,
                             prox_mu, corr, betas, eps, max_grad_norm, n, n_steps, tail, steps)
        finally:
            run.end()

    def _run(self, X, y, n_epoch, lr, batch_size, momentum, weight_decay, reshuffle_each_epoch, return_device, prox_mu,
             corr, betas, eps, max_grad_norm, n, n_steps, tail, steps):
        nn.Module.train(self.model, True)
        self._set_hyper(lr, momentum, weight_decay, prox_mu=prox_mu)
        self.prox = prox_mu > 0
        self.corr = corr
        self.clip = max_grad_norm > 0
        if self.clip:
            self._set_max_norm(max_grad_norm)
        if (momentum or self.adam) and self.arena.momentum is None:
            self.arena.momentum = torch.zeros_like(self.arena.grad)
        if self.adam and self.arena.adam_v is None:
            self.arena.adam_v = torch.zeros_like(self.arena.grad)
        # every step of the run, t = 1 .. n_epoch * steps; the first ignores the stored moments (a fresh optimizer)
        table = self._adam_rows(lr, betas, eps, weight_decay, n_epoch, steps) if self.adam else None
        stream = self._aug[2] if self._aug is not None else (self._drop[2] if self._drop is not None else None)
        aug_words = self._aug_words(stream, n_epoch) if stream is not None else None
        aug_key = self._aug[:2] if self._aug is not None else None
        drop_key = self._drop[1] if self._drop is not None else None      # baked into the captured dropout kernels
        mixing = self._mix is not None and self._mix.kind is not None
        mix_table_dev = self._mix_rows(n_epoch, steps, X) if mixing else None
        mix_key = (mixing, self._mix.smoothing) if self._mix is not None else None
        # the anchor and correction pointers are baked into the captured launches; the coefficient is read from `hyper`
        # at replay
        key = (n, batch_size, tuple(X.shape[1:]), tuple(y.shape[1:]), X.data_ptr(), y.data_ptr(), bool(momentum),
               self.prox, corr.data_ptr() if corr is not None else None, self.adam, aug_key, mix_key, self.clip, drop_key)
        epoch_losses = torch.zeros(n_epoch, 2, dtype=torch.float32, device=self.device)
        grad_norms = torch.zeros(n_epoch, steps, dtype=torch.float32, device=self.device) if self.clip else None
        if self.use_graph:
            ent = self._graphs.get(key)
            if ent is None:
                rows = table[:steps].clone() if self.adam else None
                ent = self._graphs[key] = self._capture(X, y, n_steps, batch_size, rows, steps)
            perm_full = torch.randperm(n, device=self.device)
            for e in range(n_epoch):
                if reshuffle_each_epoch and e > 0:
                    perm_full = torch.randperm(n, device=self.device)
                ent["perm"].copy_(perm_full[: n_steps * batch_size])
                if self.adam:
                    ent["rows"].copy_(table[e * steps:(e + 1) * steps])
                if aug_words is not None:
                    ent["words"].copy_(aug_words[e])
                if mixing:
                    ent["mix"].copy_(mix_table_dev[e])
                self.loss_acc.zero_()
                ent["graph"].replay()
                if ent.get("graph2") is not None:
                    self.k3_join()           # the collective of the previous round must have landed from here on
                    ent["graph2"].replay()
                if tail:
                    with torch.enable_grad():
                        self._step(X, y, perm_full[n_steps * batch_size:], fuse_sgd=False,
                                   row=ent["rows"][n_steps] if self.adam else None, s0=n_steps * batch_size,
                                   words=ent["words"], mix_rows=ent["mix"], bsz=batch_size,
                                   norm=ent["norms"][n_steps:] if self.clip else None)
                epoch_losses[e].copy_(self.loss_acc)
                if self.clip:
                    grad_norms[e].copy_(ent["norms"])
        else:
            perm_full = torch.randperm(n, device=self.device)
            for e in range(n_epoch):
                if reshuffle_each_epoch and e > 0:
                    perm_full = torch.randperm(n, device=self.device)
                self.loss_acc.zero_()
                for s, idx in enumerate(torch.split(perm_full, batch_size)):
                    with torch.enable_grad():
                        self._step(X, y, idx, row=table[e * steps + s] if self.adam else None, s0=s * batch_size,
                                   words=aug_words[e] if aug_words is not None else None,
                                   mix_rows=mix_table_dev[e] if mixing else None, bsz=batch_size,
                                   norm=grad_norms[e, s:s + 1] if self.clip else None)
                epoch_losses[e].copy_(self.loss_acc)
        self.last_steps = steps
        self.grad_norms = grad_norms
        self.last_had_tail_step = bool(tail)        # a ragged eager step ran after the graph: its SGD did not emit the wire
        if self.use_graph:
            self.emitted_wire = bool(self.graph_emits_wire and not tail)
        if return_device:                     # caller reads (or forwards) the losses itself: no host sync here
            return epoch_losses
        host = epoch_losses.tolist()          # the ONLY host read of the round
        self.last_stats = {"accuracy": [h[1] / n for h in host], "steps_per_epoch": steps}
        return [h[0] / steps for h in host]


    def last_grad_norms(self) -> Optional[List[List[float]]]:
        """The pre-clip gradient norm of every step of the last run, ``[n_epoch][steps]`` (a host read); None when it
        did not clip."""
        return self.grad_norms.tolist() if self.grad_norms is not None else None


class PortableLocalSGD:
    """Same interface as :class:`GraphedLocalSGD` on plain PyTorch ops -- CPU / gloo runs of the SPMD engine
    (plumbing config, host-side logic tests).  Parameters stay views of the arena, so the session's reduce and
    broadcast work unchanged."""

    def __init__(self, model: nn.Module, arena, *, loss: str = "ce", **_unused):
        self.model, self.arena = model, arena
        self.loss_kind = loss
        self.device = arena.device
        self.last_steps = 1
        self.kernels_per_epoch = 0
        self.n_kernels_per_step = 0
        self.last_stats = {}
        self._aug_streams = AugmentStreams()
        self.grad_norms = None        # [n_epoch, steps] pre-clip gradient norms of the last run (None: no clipping)

    def run(self, X, y, n_epoch: int = 1, lr: float = 0.001, batch_size: int = 32, momentum: float = 0.0,
            weight_decay: float = 0.0, reshuffle_each_epoch: bool = False, return_device: bool = False,
            prox_mu: float = 0.0, corr: Optional[torch.Tensor] = None, optimizer: str = "sgd",
            betas: Tuple[float, float] = (0.9, 0.999), eps: float = 1e-8, augment: Optional[str] = None,
            augment_padding: int = 4, augment_seed: Optional[int] = None, augment_stream: Optional[int] = None,
            mix: Optional[str] = None, mix_alpha: float = 1.0, label_smoothing: float = 0.0,
            max_grad_norm: float = 0.0, **_ignored):
        """``prox_mu > 0``: FedProx toward ``arena.global_w``, the global model the round started from.  ``corr``:
        SCAFFOLD's correction ``c - c_i`` (fp32, indexed like the arena's parameters), added to every gradient.
        ``optimizer="adamw"``: a fresh ``torch.optim.AdamW(lr, betas, eps, weight_decay)`` instead of SGD.
        ``augment``, ``mix``, ``label_smoothing``: as in :meth:`GraphedLocalSGD.run`, through the host references.
        ``max_grad_norm > 0``: ``clip_grad_norm_(parameters, max_grad_norm)`` right after every backward, before the
        FedProx and SCAFFOLD terms are added."""
        criterion = _loss_fn(self.loss_kind)
        prox_mu = check_prox_mu(prox_mu)
        max_grad_norm = check_max_grad_norm(max_grad_norm)
        _check_corr(corr, self.arena)
        adam = check_optimizer(optimizer, momentum, prox_mu=prox_mu, corr=corr)
        mixc = _mix_setup(mix, mix_alpha, label_smoothing, self.loss_kind)
        aug = _augment_setup(self._aug_streams, X, augment, augment_padding, augment_seed, augment_stream, mixc)
        drop = _dropout_setup(self.model, self._aug_streams, aug, augment_seed, augment_stream)
        n = X.shape[0]
        batch_size = min(batch_size, n)
        if drop is not None:
            drop[0].begin(drop[1], drop[2], -(-n // batch_size), n_epoch, self.model.n_dropout_sites)
        try:
            return self._run(X, y, n_epoch, lr, batch_size, momentum, weight_decay, reshuffle_each_epoch,
                             return_device, prox_mu, corr, betas, eps, max_grad_norm, criterion, adam, mixc, aug, drop)
        finally:
            if drop is not None:
                drop[0].end()

    def _run(self, X, y, n_epoch, lr, batch_size, momentum, weight_decay, reshuffle_each_epoch, return_device, prox_mu,
             corr, betas, eps, max_grad_norm, criterion, adam, mixc, aug, drop):
        n = X.shape[0]
        nn.Module.train(self.model, True)
        a = self.arena
        if prox_mu > 0 and a.global_w is None:
            raise ValueError("prox_mu > 0 needs the arena's global copy (ParamArena(keep_global=True))")
        params, anchors, corrs = [], [], []
        for name, p in self.model.named_parameters():
            params.append(p)
            anchors.append(a._view(a.global_w, a.slots[name]) if prox_mu > 0 else None)
            corrs.append(a._view(corr, a.slots[name]) if corr is not None else None)
        if adam:
            betas, eps = check_adamw(betas, eps)
            opt = torch.optim.AdamW(params, lr=lr, betas=betas, eps=eps, weight_decay=weight_decay)
        else:
            opt = torch.optim.SGD(params, lr=lr, momentum=momentum, weight_decay=weight_decay)
        perm = torch.randperm(n)
        out = torch.zeros(n_epoch, 2, dtype=torch.float32)
        norms = torch.zeros(n_epoch, -(-n // batch_size), dtype=torch.float32) if max_grad_norm > 0 else None
        steps = 1
        for e in range(n_epoch):
            if reshuffle_each_epoch and e > 0:
                perm = torch.randperm(n)
            batches = torch.split(perm, batch_size)
            steps = len(batches)
            rows = _host_mix_rows(mixc, aug, X, e, steps)
            for b, idx in enumerate(batches):
                opt.zero_grad(set_to_none=True)
                if drop is not None:
                    drop[0].at(e, b)
                xb = _host_batch(X, idx, aug, e, b * batch_size)
                tgt = y[idx]
                if mixc is not None:
                    xb, soft = mix_batch_reference(xb, tgt, rows[b] if rows is not None else None, mixc.smoothing)
                pred = self.model(xb)
                if pred.shape != tgt.shape and tgt.dtype.is_floating_point:
                    tgt = tgt.reshape(pred.shape)
                if mixc is not None:
                    loss = soft_cross_entropy(pred, soft)
                else:
                    loss = criterion(pred.float() if tgt.dtype.is_floating_point else pred, tgt)
                loss.backward()
                if norms is not None:
                    norms[e, b] = _clip_grads(params, max_grad_norm)
                if prox_mu > 0:
                    _add_prox_term(params, anchors, prox_mu)
                if corr is not None:
                    with torch.no_grad():
                        for p, cv in zip(params, corrs):     # a parameter without a gradient still moves by corr
                            p.grad = cv.clone() if p.grad is None else p.grad.add_(cv)
                opt.step()
                out[e, 0] += float(loss.detach())
                if mixc is not None:
                    out[e, 1] += float(soft_hits(pred, soft))
                elif not tgt.dtype.is_floating_point:
                    out[e, 1] += float((pred.argmax(-1) == tgt).sum())
        self.last_steps = steps
        self.grad_norms = norms
        if self.arena.theta_bf16 is not None:
            self.arena.sync_shadow()
        if return_device:
            return out
        host = out.tolist()
        self.last_stats = {"accuracy": [h[1] / n for h in host], "steps_per_epoch": steps}
        return [h[0] / steps for h in host]

    def last_grad_norms(self) -> Optional[List[List[float]]]:
        """The pre-clip gradient norm of every step of the last run, ``[n_epoch][steps]``; None when it did not clip."""
        return self.grad_norms.tolist() if self.grad_norms is not None else None

    def evaluate(self, X, y, batch_size: int = 512):
        """Same contract as :meth:`GraphedLocalSGD.evaluate` on plain PyTorch ops."""
        n = X.shape[0]
        was_training = self.model.training
        nn.Module.train(self.model, False)
        loss_sum = correct = 0.0
        try:
            with torch.no_grad():
                for xb, yb in zip(torch.split(X, max(1, batch_size)), torch.split(y, max(1, batch_size))):
                    pred = self.model(xb)
                    if yb.dtype.is_floating_point:
                        per_row = max(1, pred.numel() // max(1, pred.shape[0]))
                        loss_sum += float(((pred.float() - yb.reshape(pred.shape).float()) ** 2).sum()) / per_row
                    else:
                        loss_sum += float(nn.functional.cross_entropy(pred.float(), yb, reduction="sum"))
                        correct += float((pred.argmax(-1) == yb).sum())
        finally:
            nn.Module.train(self.model, was_training)
        return loss_sum, correct, float(n)
