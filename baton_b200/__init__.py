"""baton_b200 -- a Hopper-native federated-learning engine with the
capabilities and API of mynameisfiber/baton.

Layers (SURVEY.md section 1 / 7.1):
  control/   aiohttp control plane: Manager, Experiment, ClientManager, UpdateManager, ExperimentWorker
  parallel/  data planes (http | fused NVLink | nccl), flat symmetric arena, fused FedAvg collective
  ops/       hand-written sm_90a kernels (wgmma GEMM, conv, BatchNorm, LayerNorm, losses, fused SGD)
  models/    demo linear model, MLP, ResNet-18/50, BERT-base built on ``ops``
  data/      synthetic IID / label-skew / Dirichlet shards
  utils/     asyncio helpers, key minting, JSON scrubbing, progress, clock seam
"""
from .control import (ClientManager, Experiment, ExperimentWorker, Manager, UpdateException,
                      UpdateInProgress, UpdateManager, UpdateNotInProgress)
from .utils import EpochProgress, PeriodicTask, ensure_no_collision, json_clean, random_key

__version__ = "0.1.0"

__all__ = [
    "Manager", "Experiment", "ClientManager", "UpdateManager", "ExperimentWorker",
    "UpdateException", "UpdateInProgress", "UpdateNotInProgress",
    "EpochProgress", "PeriodicTask", "ensure_no_collision", "json_clean", "random_key",
]
