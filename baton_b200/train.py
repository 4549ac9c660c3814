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
"""
from __future__ import annotations

import contextlib
import gc
from collections import OrderedDict
from typing import Callable, List, Optional, Tuple

import torch
from torch import nn

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


OPTIMIZERS = ("sgd", "adamw")


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
    """True for ``"adamw"``, False for ``"sgd"``; ``ValueError`` for another name, or for AdamW together with
    momentum, Nesterov, FedProx or SCAFFOLD (terms of the SGD step)."""
    if optimizer not in OPTIMIZERS:
        raise ValueError("optimizer must be one of {}, got {!r}".format(OPTIMIZERS, optimizer))
    if optimizer != "adamw":
        return False
    if momentum or nesterov:
        raise ValueError("momentum / nesterov are SGD options; AdamW keeps its own moments (betas)")
    if prox_mu > 0:
        raise ValueError("AdamW with FedProx (prox_mu > 0) is not supported")
    if corr is not None:
        raise ValueError("AdamW with SCAFFOLD is not supported: its control-variate update assumes SGD steps")
    return True


def _add_prox_term(params, anchors, prox_mu: float) -> None:
    """FedProx: ``grad += prox_mu * (w - anchor)`` before the optimizer step (what the reference implementation does)."""
    with torch.no_grad():
        for p, a in zip(params, anchors):
            if p.grad is not None:
                p.grad.add_(p.detach() - a, alpha=prox_mu)


def _check_corr(corr, prox_mu: float, arena) -> None:
    if corr is None:
        return
    if prox_mu > 0:
        raise ValueError("SCAFFOLD's correction and FedProx's proximal term are exclusive")
    if corr.dtype != torch.float32 or not corr.is_contiguous() or corr.numel() < arena.n_param:
        raise ValueError("corr must be a contiguous fp32 buffer covering the arena's parameters")


def run_local_sgd(model: nn.Module, X: torch.Tensor, y: torch.Tensor, *, n_epoch: int = 32,
                  lr: float = 0.001, batch_size: int = 32, momentum: float = 0.0,
                  weight_decay: float = 0.0, loss: "str | Callable" = "mse",
                  verbose: bool = False, reshuffle_each_epoch: bool = False,
                  generator: Optional[torch.Generator] = None, prox_mu: float = 0.0, optimizer: str = "sgd",
                  betas: Tuple[float, float] = (0.9, 0.999), eps: float = 1e-8) -> List[float]:
    """Portable local SGD; returns the per-epoch mean loss.  ``prox_mu > 0``: FedProx, anchored on the parameters as
    they are on entry -- the global model the worker has just loaded.  ``optimizer="adamw"``: a fresh
    ``torch.optim.AdamW(lr, betas, eps, weight_decay)`` instead of SGD."""
    criterion = _loss_fn(loss)
    prox_mu = check_prox_mu(prox_mu)
    adam = check_optimizer(optimizer, momentum, prox_mu=prox_mu)
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
        batch_iter = EpochProgress(epoch, torch.split(idxs, batch_size), verbose=verbose)
        for batch_idxs in batch_iter:
            optimizer.zero_grad(set_to_none=True)
            output = model(X[batch_idxs])
            target = y[batch_idxs]
            if output.shape != target.shape and target.dtype.is_floating_point:
                target = target.reshape(output.shape)  # (N,) vs (N,1) -- quirk 13
            loss_batch = criterion(output, target)
            batch_iter.update_loss(loss_batch)
            loss_batch.backward()
            if anchors is not None:
                _add_prox_term(params, anchors, prox_mu)
            optimizer.step()
        loss_history.append(batch_iter.loss)
    return loss_history


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
        self.hyper = torch.zeros(5, dtype=torch.float32, device=dev)   # [lr, momentum, wd, dampening, prox_mu]
        self.prox = False             # FedProx: every SGD kernel of the step reads the anchor arena.global_w
        self.corr = None              # SCAFFOLD: every SGD kernel of the step reads this correction c - c_i
        self.adam = False             # AdamW: every optimizer kernel of the step reads its step row and arena.adam_v
        self._adam_table = (None, None)   # (host key, device [n_epoch * steps, ADAMW_ROW] rows of the run)
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
    def _loss(self, out, yb):
        if self.loss_kind in ("ce", "cross_entropy"):
            loss, stats = self.bnn.cross_entropy(out, yb)
            return loss, stats
        loss = self.bnn.mse_loss(out, yb)
        return loss, torch.stack([loss.detach(), torch.zeros_like(loss.detach())])

    def _gather(self, X, y, idx):
        F = self.F
        xb = F.gather_rows(X, idx)
        yb = F.gather_rows(y, idx) if y.dtype == torch.int64 and y.dim() == 1 else y.index_select(0, idx)
        return xb, yb

    def _step(self, X, y, idx, batch=None, emit_wire=False, fuse_sgd=True, row=None):
        """One SGD step on ``X[idx], y[idx]`` (or on the already gathered ``batch``).  ``emit_wire``: last step of
        an epoch -- the optimizer kernel also writes the upload copy for the round-end collective (``self.pack``).
        ``fuse_sgd=False``: no optimizer epilogue in the weight-gradient GEMMs (one optimizer pass over the arena).
        ``row``: with AdamW, the device row of this step's coefficients (``F.adamw_rows``)."""
        F = self.F
        xb, yb = batch if batch is not None else self._gather(X, y, idx)
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
                # the split-K = 1 convolution weight gradients apply SGD in their GEMM epilogue; one launch covers the rest
                with self.bnn.SGD_EPI.open(a, hyper, self.nesterov, prox=self.prox, corr=self.corr,
                                           adam_v=adam_v) as epi:
                    explicit(xb, yb, loss_acc=self.loss_acc, after_first_gemm=self._first_gemm_hook)
                F.fused_sgd_segments(a.theta, a.grad, hyper, self._segment_table(epi.fused, epi.nograd),
                                     a.momentum, bf, nesterov=self.nesterov, prox_anchor=anchor, corr=self.corr,
                                     adam_v=adam_v)
                self.emitted_wire = False
                return
            explicit(xb, yb, loss_acc=self.loss_acc, after_first_gemm=self._first_gemm_hook)
            stats = None
        else:
            out = self.model(xb)
            loss, stats = self._loss(out, yb)
            loss.backward()
            self.bnn.WGRAD.join()      # weight-gradient GEMMs run on a side stream; they must land before the step
        # one optimizer pass over the whole arena; the epoch's last step also emits the upload copy
        pack = self.pack if emit_wire else None
        F.fused_sgd(a.theta[: a.n_param], a.grad, hyper, a.momentum,
                    bf[: a.n_param] if bf is not None else None, zero_grad=True, nesterov=self.nesterov, pack=pack,
                    prox_anchor=anchor[: a.n_param] if anchor is not None else None,
                    corr=self.corr[: a.n_param] if self.corr is not None else None, adam_v=adam_v)
        self.emitted_wire = pack is not None
        if stats is not None:
            self.loss_acc.add_(stats)

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
            self.hyper.copy_(torch.tensor(vals, dtype=torch.float32))
            self._hyper_host = vals

    def _adam_rows(self, lr, betas, eps, weight_decay, n_epoch, steps):
        """Device ``[n_epoch * steps, ADAMW_ROW]`` AdamW coefficients of every local step of a run (step ``t`` counts
        across epochs); copied to the device only when they change."""
        key = (float(lr), tuple(betas), float(eps), float(weight_decay), n_epoch, steps)
        if self._adam_table[0] != key:
            rows = self.F.adamw_rows(lr, betas, eps, weight_decay, 1, n_epoch * steps)
            self._adam_table = (key, rows.to(self.device))
        return self._adam_table[1]

    # -------------------------------------------------------------- epoch graph
    def _capture(self, X, y, n_steps, batch_size, rows=None):
        """``rows``: with AdamW, the device row buffer captured step ``s`` reads row ``s`` of (holding the first
        epoch's rows, which the warm-up steps use too); kept in the returned entry."""
        perm = torch.zeros(n_steps * batch_size, dtype=torch.int64, device=self.device)
        perm.copy_(torch.arange(n_steps * batch_size, device=self.device) % X.shape[0])
        side = torch.cuda.Stream(device=self.device)
        side.wait_stream(torch.cuda.current_stream(self.device))
        with torch.cuda.stream(side):   # warm-up outside capture (allocator, lazy init, autograd)
            # hyper lr=0 during warm-up/capture would still move BN statistics; save/restore the state
            snap = self.arena.theta.clone()
            snap_i = self.arena.int_arena.clone()
            snap_m = self.arena.momentum.clone() if self.arena.momentum is not None else None
            for _ in range(2):
                self._step(X, y, perm[:batch_size], row=rows[0] if rows is not None else None)
        torch.cuda.current_stream(self.device).wait_stream(side)
        torch.cuda.synchronize(self.device)
        from .ops._ext import total_launches
        graph = torch.cuda.CUDAGraph()
        graph2 = None
        c0 = total_launches()

        def body():
            # the epoch's batches are gathered by ONE launch pair (a permuted copy of the shard, 25 MB for the
            # flagship config) instead of two latency-bound gathers at the head of every step
            Xp, yp = self._gather(X, y, perm)
            for s in range(n_steps):
                self._step(X, y, None, batch=(Xp[s * batch_size:(s + 1) * batch_size],
                                              yp[s * batch_size:(s + 1) * batch_size]),
                           emit_wire=(s == n_steps - 1 and self.pack is not None),
                           row=rows[s] if rows is not None else None)
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
        return {"graph": graph, "graph2": graph2, "perm": perm, "X": X, "y": y, "rows": rows}

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
                explicit = False
            else:
                table, size = fold
                out = torch.zeros(size, dtype=torch.float32, device=self.device)
                self._fold = (table, out)
                self.model.eval_bn_table = out
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
            betas: Tuple[float, float] = (0.9, 0.999), eps: float = 1e-8, **_ignored):
        """``prox_mu > 0``: FedProx toward ``arena.global_w``, the global model the round started from.  ``corr``:
        SCAFFOLD's correction ``c - c_i`` (fp32 device buffer of ``arena.n_param`` elements), added to every step's
        gradient; it is read at replay, so the caller may rewrite it between runs.  ``optimizer="adamw"``: the steps of
        a fresh ``torch.optim.AdamW(lr, betas, eps, weight_decay)`` instead of SGD."""
        assert X.is_cuda, "GraphedLocalSGD needs a device-resident shard"
        prox_mu = check_prox_mu(prox_mu)
        if prox_mu > 0 and self.arena.global_w is None:
            raise ValueError("prox_mu > 0 needs the arena's global copy (ParamArena(keep_global=True))")
        _check_corr(corr, prox_mu, self.arena)
        self.adam = check_optimizer(optimizer, momentum, self.nesterov, prox_mu, corr)
        if self.adam:
            betas, eps = check_adamw(betas, eps)
        nn.Module.train(self.model, True)
        n = X.shape[0]
        batch_size = min(batch_size, n)
        n_steps = n // batch_size
        tail = n - n_steps * batch_size
        steps = n_steps + (1 if tail else 0)
        self._set_hyper(lr, momentum, weight_decay, prox_mu=prox_mu)
        self.prox = prox_mu > 0
        self.corr = corr
        if (momentum or self.adam) and self.arena.momentum is None:
            self.arena.momentum = torch.zeros_like(self.arena.grad)
        if self.adam and self.arena.adam_v is None:
            self.arena.adam_v = torch.zeros_like(self.arena.grad)
        # every step of the run, t = 1 .. n_epoch * steps; the first ignores the stored moments (a fresh optimizer)
        table = self._adam_rows(lr, betas, eps, weight_decay, n_epoch, steps) if self.adam else None
        # the anchor and correction pointers are baked into the captured launches; the coefficient is read from `hyper`
        # at replay
        key = (n, batch_size, tuple(X.shape[1:]), tuple(y.shape[1:]), X.data_ptr(), y.data_ptr(), bool(momentum),
               self.prox, corr.data_ptr() if corr is not None else None, self.adam)
        epoch_losses = torch.zeros(n_epoch, 2, dtype=torch.float32, device=self.device)
        if self.use_graph:
            ent = self._graphs.get(key)
            if ent is None:
                rows = table[:steps].clone() if self.adam else None
                ent = self._graphs[key] = self._capture(X, y, n_steps, batch_size, rows)
            perm_full = torch.randperm(n, device=self.device)
            for e in range(n_epoch):
                if reshuffle_each_epoch and e > 0:
                    perm_full = torch.randperm(n, device=self.device)
                ent["perm"].copy_(perm_full[: n_steps * batch_size])
                if self.adam:
                    ent["rows"].copy_(table[e * steps:(e + 1) * steps])
                self.loss_acc.zero_()
                ent["graph"].replay()
                if ent.get("graph2") is not None:
                    self.k3_join()           # the collective of the previous round must have landed from here on
                    ent["graph2"].replay()
                if tail:
                    with torch.enable_grad():
                        self._step(X, y, perm_full[n_steps * batch_size:], fuse_sgd=False,
                                   row=ent["rows"][n_steps] if self.adam else None)
                epoch_losses[e].copy_(self.loss_acc)
        else:
            perm_full = torch.randperm(n, device=self.device)
            for e in range(n_epoch):
                if reshuffle_each_epoch and e > 0:
                    perm_full = torch.randperm(n, device=self.device)
                self.loss_acc.zero_()
                for s, idx in enumerate(torch.split(perm_full, batch_size)):
                    with torch.enable_grad():
                        self._step(X, y, idx, row=table[e * steps + s] if self.adam else None)
                epoch_losses[e].copy_(self.loss_acc)
        self.last_steps = steps
        self.last_had_tail_step = bool(tail)        # a ragged eager step ran after the graph: its SGD did not emit the wire
        if self.use_graph:
            self.emitted_wire = bool(self.graph_emits_wire and not tail)
        if return_device:                     # caller reads (or forwards) the losses itself: no host sync here
            return epoch_losses
        host = epoch_losses.tolist()          # the ONLY host read of the round
        self.last_stats = {"accuracy": [h[1] / n for h in host], "steps_per_epoch": steps}
        return [h[0] / steps for h in host]


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

    def run(self, X, y, n_epoch: int = 1, lr: float = 0.001, batch_size: int = 32, momentum: float = 0.0,
            weight_decay: float = 0.0, reshuffle_each_epoch: bool = False, return_device: bool = False,
            prox_mu: float = 0.0, corr: Optional[torch.Tensor] = None, optimizer: str = "sgd",
            betas: Tuple[float, float] = (0.9, 0.999), eps: float = 1e-8, **_ignored):
        """``prox_mu > 0``: FedProx toward ``arena.global_w``, the global model the round started from.  ``corr``:
        SCAFFOLD's correction ``c - c_i`` (fp32, indexed like the arena's parameters), added to every gradient.
        ``optimizer="adamw"``: a fresh ``torch.optim.AdamW(lr, betas, eps, weight_decay)`` instead of SGD."""
        criterion = _loss_fn(self.loss_kind)
        prox_mu = check_prox_mu(prox_mu)
        _check_corr(corr, prox_mu, self.arena)
        adam = check_optimizer(optimizer, momentum, prox_mu=prox_mu, corr=corr)
        n = X.shape[0]
        batch_size = min(batch_size, n)
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
        steps = 1
        for e in range(n_epoch):
            if reshuffle_each_epoch and e > 0:
                perm = torch.randperm(n)
            batches = torch.split(perm, batch_size)
            steps = len(batches)
            for idx in batches:
                opt.zero_grad(set_to_none=True)
                pred = self.model(X[idx])
                tgt = y[idx]
                if pred.shape != tgt.shape and tgt.dtype.is_floating_point:
                    tgt = tgt.reshape(pred.shape)
                loss = criterion(pred.float() if tgt.dtype.is_floating_point else pred, tgt)
                loss.backward()
                if prox_mu > 0:
                    _add_prox_term(params, anchors, prox_mu)
                if corr is not None:
                    with torch.no_grad():
                        for p, cv in zip(params, corrs):     # a parameter without a gradient still moves by corr
                            p.grad = cv.clone() if p.grad is None else p.grad.add_(cv)
                opt.step()
                out[e, 0] += float(loss.detach())
                if not tgt.dtype.is_floating_point:
                    out[e, 1] += float((pred.argmax(-1) == tgt).sum())
        self.last_steps = steps
        if self.arena.theta_bf16 is not None:
            self.arena.sync_shadow()
        if return_device:
            return out
        host = out.tolist()
        self.last_stats = {"accuracy": [h[1] / n for h in host], "steps_per_epoch": steps}
        return [h[0] / steps for h in host]

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
