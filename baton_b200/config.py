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
    model: str = "lineartest"          # lineartest | mlp2 | resnet18 | resnet50 | resnet18_gn | resnet50_gn | bert_base |
    #                                    vit_tiny | vit_small
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
    augment: str = "none"              # local-training augmentation: none | crop | flip | crop_flip (NHWC image shards)
    augment_padding: int = 4           # zero padding of the random crop, pixels on each side
    mix: str = "none"                  # batch mixing: none | mixup | cutmix | mixup_cutmix (NHWC images, cross-entropy)
    mix_alpha: float = 1.0             # lambda ~ Beta(mix_alpha, mix_alpha), one per batch
    label_smoothing: float = 0.0       # soft-target smoothing eps in [0, 1) of the training cross-entropy
    max_grad_norm: float = 0.0         # clip_grad_norm_ of every local step's gradient to this 2-norm (0: off)
    dropout: float = 0.0               # BERT: hidden and attention-probability dropout (the classifier follows hidden)
    lora_r: int = 0                    # BERT: LoRA rank, 8 | 16 | 32 | 64 (0: full fine-tuning)
    lora_alpha: float = 16.0           # LoRA scale alpha / r
    lora_targets: str = "query,value"  # comma-separated subset of query, key, value, attn_out, ffn_in, ffn_out
    lora_freeze_a: bool = False        # FFA-LoRA: A stays frozen, only B and the classifier train
    dp_clip: float = 0.0               # DP-FedAvg: L2 clip norm of a client's update (0: DP off)
    dp_noise_multiplier: float = 0.0   # DP-FedAvg: noise std on the sum of clipped updates, in units of dp_clip
    dp_delta: float = 1e-5             # DP-FedAvg: delta of the (epsilon, delta) the manager reports
    dp_seed: Optional[int] = None      # DP-FedAvg noise key (None: secret random; an explicit key is for tests only)
    aggregator: str = "mean"           # mean | median | trimmed_mean (coordinate-wise) | krum (Multi-Krum); unweighted
    trim_ratio: float = 0.1            # trimmed_mean: fraction trimmed at each end, 0 <= beta < 0.5
    krum_f: int = 0                    # krum: Byzantine clients assumed (needs >= 2f + 3 participants per round)
    krum_m: Optional[int] = None       # krum: clients kept (None: participants - f; 1: classic Krum)
    server_opt: str = "none"           # server optimizer on the aggregate: none | avgm | adagrad | yogi | adam
    server_lr: Optional[float] = None  # server learning rate (required with a server optimizer; no default)
    server_beta1: float = 0.9          # server optimizer decays and adaptivity floor (Reddi et al.'s defaults)
    server_beta2: float = 0.99
    server_tau: float = 1e-3
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
        from .train import check_adamw, check_max_grad_norm, check_prox_mu
        check_prox_mu(self.prox_mu)
        check_max_grad_norm(self.max_grad_norm)
        check_adamw((self.adam_beta1, self.adam_beta2), self.adam_eps)
        from .data.augment import check_augment
        check_augment(self.augment, self.augment_padding)
        from .data.mix import check_mix
        check_mix(self.mix, self.mix_alpha, self.label_smoothing)
        from .data.dropout import check_dropout
        check_dropout(self.dropout, "dropout")
        if self.dropout > 0.0 and self.model != "bert_base":
            raise ValueError("dropout applies to the BERT models only, not {!r}".format(self.model))
        if self.lora_r:
            if self.model != "bert_base":
                raise ValueError("LoRA applies to bert_base only, not {!r}".format(self.model))
            self.lora_config()
        from .parallel.dp import check_dp
        check_dp(self.dp_clip, self.dp_noise_multiplier)
        if not (0.0 < float(self.dp_delta) < 1.0):
            raise ValueError("dp_delta must lie in (0, 1), got {!r}".format(self.dp_delta))
        from .parallel.robust import check_aggregator
        self.trim_ratio = check_aggregator(self.aggregator, self.trim_ratio)
        if self.aggregator == "krum":
            from .parallel.features import round_plan
            from .parallel.robust import check_krum, check_krum_participants
            check_krum(self.krum_f, self.krum_m)
            check_krum_participants(round_plan(self.clients, self.logical_clients, self.sample_k)[0], self.krum_f)
        self.server_opt_config()          # validates kind, lr, betas and tau
        from .parallel.features import check_features
        check_features(dp=float(self.dp_clip) > 0.0, robust=self.aggregator != "mean",
                       server_opt=self.server_opt != "none",
                       plane="seated" if self.backend in ("fused", "nccl") else "http", optimizer=self.optimizer,
                       momentum=self.momentum, prox_mu=float(self.prox_mu), frozen=bool(self.lora_r))

    def lora_config(self):
        """The :class:`~baton_b200.models.bert.LoraConfig` of these fields, or None (``lora_r == 0``)."""
        if not self.lora_r:
            return None
        from .models.bert import LoraConfig
        return LoraConfig(self.lora_r, self.lora_alpha, tuple(t.strip() for t in self.lora_targets.split(",")),
                          self.lora_freeze_a)

    def train_kwargs(self) -> dict:
        """Local-training keyword arguments of a worker (``FederatedModule.local_train``)."""
        kw = {"lr": self.lr, "batch_size": self.batch_size, "prox_mu": self.prox_mu}
        if self.optimizer != "sgd":
            kw.update(optimizer=self.optimizer, betas=(self.adam_beta1, self.adam_beta2), eps=self.adam_eps)
        if self.augment != "none":
            kw.update(augment=self.augment, augment_padding=self.augment_padding)
        if self.mix != "none":
            kw.update(mix=self.mix, mix_alpha=self.mix_alpha)
        if self.label_smoothing != 0.0:
            kw.update(label_smoothing=self.label_smoothing)
        if self.max_grad_norm > 0.0:
            kw.update(max_grad_norm=self.max_grad_norm)
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
        return RobustConfig(self.aggregator, self.trim_ratio, self.krum_f, self.krum_m)

    def server_opt_config(self):
        """The :class:`~baton_b200.parallel.server_opt.ServerOptConfig` of these fields, or None (``"none"``)."""
        if self.server_opt == "none":
            return None
        from .parallel.server_opt import ServerOptConfig
        return ServerOptConfig(self.server_opt, self.server_lr, self.server_beta1, self.server_beta2, self.server_tau)

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
            if f.name in ("sample_k", "dp_seed", "krum_m"):
                typ = int
            if f.name in ("round_timeout", "server_lr"):
                typ = float
            if f.name in ("checkpoint_dir",):
                typ = str
            if typ is bool:
                typ = lambda v: v.lower() in ("1", "true", "yes")    # noqa: E731
            parser.add_argument(flag, dest=f.name, type=typ, default=default)

    @classmethod
    def from_args(cls, ns: argparse.Namespace) -> "FederationConfig":
        return cls(**{f.name: getattr(ns, f.name) for f in fields(cls) if hasattr(ns, f.name)})
