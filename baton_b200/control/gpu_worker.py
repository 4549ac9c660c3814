"""GPU-seated federated client: the reference worker contract on the NVLink data plane.

``GpuExperimentWorker`` is an :class:`ExperimentWorker` (reference worker.py:12-127: register,
heartbeat, ``round_start`` -> local training -> ``report_update``) whose model lives in a flat
parameter arena on one GPU and whose uploads/downloads never touch HTTP: the POSTs carry metadata
only and the round-end reduce + broadcast is the fused NVLink kernel, launched on every seat when
the manager sends the aggregation plan (``POST /{name}/aggregate``).

One process per GPU; ``torch.distributed`` (NCCL) is initialised by the launcher and is used only to
bootstrap the symmetric-memory rendezvous.
"""
from __future__ import annotations

from typing import Callable, Optional, Tuple

import torch
from aiohttp import web

from ..parallel.arena import ParamArena
from ..parallel.fedavg import FedAvgSession, NcclSession
from ..train import GraphedLocalSGD
from ..utils.aio import run_blocking
from .worker import ExperimentWorker


class EvaluatingSeat:
    """``POST /{name}/evaluate`` of a seat that holds the global model: evaluates it on the seat's held-out shard
    (``eval_shard_fn() -> (X, y)``) with ``self.trainer.evaluate`` on the training thread, off the event loop, and
    answers JSON ``{n_samples, loss_sum, correct}``.  501 when the seat has no held-out data."""

    eval_shard_fn: Optional[Callable[[], Tuple[torch.Tensor, torch.Tensor]]] = None
    eval_batch_size = 512

    def register_handlers(self) -> None:
        super().register_handlers()
        self.app.router.add_post("/{}/evaluate".format(self.name), self.evaluate)

    async def evaluate(self, request: web.Request) -> web.Response:
        if not self._credentials_ok(request):
            return web.json_response({"err": "Wrong Client"}, status=404)
        if self.eval_shard_fn is None:
            return web.json_response({"err": "No Evaluation Data"}, status=501)
        loss_sum, correct, n = await run_blocking(self._evaluate_blocking, executor=self._executor)
        return web.json_response({"n_samples": n, "loss_sum": loss_sum, "correct": correct})

    def _evaluate_blocking(self):
        X, y = self.eval_shard_fn()
        return self.trainer.evaluate(X, y, batch_size=self.eval_batch_size)


class GpuExperimentWorker(EvaluatingSeat, ExperimentWorker):
    def __init__(self, app, model, manager: str, *, device, shard_fn: Callable[[], Tuple[torch.Tensor, torch.Tensor]],
                 backend: str = "fused", group=None, loss: str = "ce", wire_dtype: str = "bf16",
                 momentum: float = 0.0, use_graph: bool = True, n_ctas: int = 64,
                 eval_shard_fn: Optional[Callable[[], Tuple[torch.Tensor, torch.Tensor]]] = None,
                 eval_batch_size: int = 512, robust=None, **kwargs):
        """``eval_shard_fn`` (optional): ``() -> (X, y)``, this seat's held-out shard for ``POST /{name}/evaluate``.
        ``robust`` (optional :class:`~baton_b200.parallel.robust.RobustConfig`): the session's aggregator.  A seat of a
        Krum experiment needs it, because a fused Krum session allocates its distance page at construction."""
        self.device = torch.device(device)
        self.eval_shard_fn, self.eval_batch_size = eval_shard_fn, eval_batch_size
        self._eval_stage = None
        torch.cuda.set_device(self.device)          # the constructing thread (usually the event-loop thread)
        self.arena = ParamArena(model, self.device, momentum=momentum > 0)
        if hasattr(model, "build_workspace"):
            model.build_workspace(self.device)
        self.trainer = GraphedLocalSGD(model, self.arena, loss=loss, use_graph=use_graph)
        model._graphed_trainer = self.trainer
        Session = {"fused": FedAvgSession, "nccl": NcclSession}[backend]
        self.fed_session = Session(self.arena, group, wire_dtype=wire_dtype, n_ctas=n_ctas, robust=robust)
        self.shard_fn = shard_fn
        self._stage = None
        train_kwargs = dict(kwargs.pop("train_kwargs", None) or {})
        if momentum:
            train_kwargs.setdefault("momentum", momentum)
        super().__init__(app, model, manager, dataplane=backend, session=self.fed_session,
                         train_kwargs=train_kwargs, **kwargs)

    def get_data(self):
        """Private shard of this round, resident on the GPU.  Host tensors returned by ``shard_fn``
        are copied into persistent staging buffers so the captured epoch graph stays valid."""
        X, y = self.shard_fn()
        if not X.is_cuda:
            if self._stage is None or self._stage[0].shape != X.shape:
                self._stage = (torch.empty(X.shape, dtype=X.dtype, device=self.device),
                               torch.empty(y.shape, dtype=y.dtype, device=self.device))
            self._stage[0].copy_(X, non_blocking=True)
            self._stage[1].copy_(y, non_blocking=True)
            X, y = self._stage
        return (X, y), int(X.shape[0])

    def _evaluate_blocking(self):
        """Held-out shards from the host are copied into their own persistent buffers (the captured evaluation
        graph keeps their addresses; the training buffers are left alone)."""
        X, y = self.eval_shard_fn()
        if not X.is_cuda:
            if self._eval_stage is None or self._eval_stage[0].shape != X.shape:
                self._eval_stage = (torch.empty(X.shape, dtype=X.dtype, device=self.device),
                                    torch.empty(y.shape, dtype=y.dtype, device=self.device))
            self._eval_stage[0].copy_(X, non_blocking=True)
            self._eval_stage[1].copy_(y, non_blocking=True)
            X, y = self._eval_stage
        return self.trainer.evaluate(X, y, batch_size=self.eval_batch_size)
