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

from typing import Callable, Tuple

import torch

from ..parallel.arena import ParamArena
from ..parallel.fedavg import FedAvgSession, NcclSession
from ..train import GraphedLocalSGD
from .worker import ExperimentWorker


class GpuExperimentWorker(ExperimentWorker):
    def __init__(self, app, model, manager: str, *, device, shard_fn: Callable[[], Tuple[torch.Tensor, torch.Tensor]],
                 backend: str = "fused", group=None, loss: str = "ce", wire_dtype: str = "bf16",
                 momentum: float = 0.0, use_graph: bool = True, n_ctas: int = 64, **kwargs):
        self.device = torch.device(device)
        torch.cuda.set_device(self.device)          # the constructing thread (usually the event-loop thread)
        self.arena = ParamArena(model, self.device, momentum=momentum > 0)
        if hasattr(model, "build_workspace"):
            model.build_workspace(self.device)
        self.trainer = GraphedLocalSGD(model, self.arena, loss=loss, use_graph=use_graph)
        model._graphed_trainer = self.trainer
        Session = {"fused": FedAvgSession, "nccl": NcclSession}[backend]
        self.fed_session = Session(self.arena, group, wire_dtype=wire_dtype, n_ctas=n_ctas)
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
