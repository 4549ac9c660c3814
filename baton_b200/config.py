"""Typed configuration for federated jobs.

The reference has no config system: three positional argv (demo.py:64-66) and
constructor defaults -- ``client_ttl=300`` (manager.py:22), ``heartbeat_time=60``,
``port=8080`` (worker.py:13-14), ``n_epoch=32`` (manager.py:55), ``lr=0.001,
batch_size=32`` (demo.py:29).  Those defaults are preserved here and extended
with the knobs the benchmark configurations need.
"""
from __future__ import annotations

import argparse
import json
from dataclasses import asdict, dataclass, fields
from typing import Optional


@dataclass
class FederationConfig:
    model: str = "lineartest"          # lineartest | mlp2 | resnet18 | resnet50 | bert_base
    dtype: str = "fp32"                # fp32 | bf16 | fp8 (block-scaled mxfp8 GEMMs)
    backend: str = "http"              # http | fused | nccl
    clients: int = 2                   # physical clients (GPUs)
    logical_clients: int = 0           # >clients => time-sliced logical clients
    sample_k: Optional[int] = None     # participants per round (None = all)
    local_epochs: int = 32             # manager.py:55
    lr: float = 0.001                  # demo.py:29
    batch_size: int = 32               # demo.py:29
    momentum: float = 0.0
    weight_decay: float = 0.0
    prox_mu: float = 0.0               # FedProx proximal coefficient (0: FedAvg's plain local SGD)
    optimizer: str = "sgd"             # local optimizer: sgd | adamw (a fresh torch.optim.AdamW per client and round)
    adam_beta1: float = 0.9            # AdamW betas and eps (read only with optimizer='adamw')
    adam_beta2: float = 0.999
    adam_eps: float = 1e-8
    dp_clip: float = 0.0               # DP-FedAvg: L2 clip norm of a client's update (0: DP off)
    dp_noise_multiplier: float = 0.0   # DP-FedAvg: noise std on the sum of clipped updates, in units of dp_clip
    dp_delta: float = 1e-5             # DP-FedAvg: delta of the (epsilon, delta) the manager reports
    dp_seed: Optional[int] = None      # DP-FedAvg noise key (None: secret random; an explicit key is for tests only)
    aggregator: str = "mean"           # mean | median | trimmed_mean (coordinate-wise, unweighted over clients)
    trim_ratio: float = 0.1            # trimmed_mean: fraction trimmed at each end, 0 <= beta < 0.5
    partition: str = "iid"             # iid | label_skew | dirichlet
    alpha: float = 0.1                 # Dirichlet concentration
    samples_per_client: int = 4096
    num_classes: int = 10
    client_ttl: float = 300.0          # manager.py:22
    heartbeat_time: float = 60.0       # worker.py:14
    round_timeout: Optional[float] = None
    wire_dtype: str = "bf16"           # precision of the upload over NVLink: fp32 | bf16
    checkpoint_dir: Optional[str] = None
    seed: int = 0

    def __post_init__(self):
        if not (0.0 <= float(self.prox_mu) < float("inf")):
            raise ValueError("prox_mu must be a finite number >= 0, got {!r}".format(self.prox_mu))
        from .train import check_adamw, check_optimizer
        check_optimizer(self.optimizer, self.momentum, prox_mu=float(self.prox_mu))
        check_adamw((self.adam_beta1, self.adam_beta2), self.adam_eps)
        from .parallel.dp import check_dp
        check_dp(self.dp_clip, self.dp_noise_multiplier)
        if not (0.0 < float(self.dp_delta) < 1.0):
            raise ValueError("dp_delta must lie in (0, 1), got {!r}".format(self.dp_delta))
        from .parallel.robust import check_aggregator
        self.trim_ratio = check_aggregator(self.aggregator, self.trim_ratio)
        if self.aggregator != "mean" and float(self.dp_clip) > 0.0:
            raise ValueError("a robust aggregator with DP-FedAvg is not supported")

    def train_kwargs(self) -> dict:
        """Local-training keyword arguments of a worker (``FederatedModule.local_train``)."""
        kw = {"lr": self.lr, "batch_size": self.batch_size, "prox_mu": self.prox_mu}
        if self.optimizer != "sgd":
            kw.update(optimizer=self.optimizer, betas=(self.adam_beta1, self.adam_beta2), eps=self.adam_eps)
        return kw

    def dp_config(self):
        """The :class:`~baton_b200.parallel.dp.DPConfig` of these fields, or None when DP is off (``dp_clip == 0``)."""
        if self.dp_clip <= 0.0:
            return None
        from .parallel.dp import DPConfig
        return DPConfig(self.dp_clip, self.dp_noise_multiplier, seed=self.dp_seed)

    def robust_config(self):
        """The :class:`~baton_b200.parallel.robust.RobustConfig` of these fields, or None for the mean."""
        if self.aggregator == "mean":
            return None
        from .parallel.robust import RobustConfig
        return RobustConfig(self.aggregator, self.trim_ratio)

    def to_json(self) -> str:
        return json.dumps(asdict(self), sort_keys=True)

    @classmethod
    def from_json(cls, text: str) -> "FederationConfig":
        known = {f.name for f in fields(cls)}
        data = json.loads(text)
        unknown = set(data) - known
        if unknown:
            raise ValueError("unknown config keys: {}".format(sorted(unknown)))
        return cls(**data)

    @classmethod
    def add_arguments(cls, parser: argparse.ArgumentParser) -> None:
        for f in fields(cls):
            flag = "--" + f.name.replace("_", "-")
            default = f.default
            typ = type(default) if default is not None else None
            if f.name in ("sample_k", "dp_seed"):
                typ = int
            if f.name in ("round_timeout",):
                typ = float
            if f.name in ("checkpoint_dir",):
                typ = str
            parser.add_argument(flag, dest=f.name, type=typ, default=default)

    @classmethod
    def from_args(cls, ns: argparse.Namespace) -> "FederationConfig":
        return cls(**{f.name: getattr(ns, f.name) for f in fields(cls) if hasattr(ns, f.name)})
