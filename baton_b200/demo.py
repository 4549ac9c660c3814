"""Command-line entry point.

Parity target: reference demo.py:62-77 --
``python demo.py {manager|worker} <manager host:port> <listen port>`` builds an
aiohttp application with either a ``Manager`` holding the example model or an
example worker with a synthetic private shard, then ``web.run_app``.  The three
positionals are unchanged (the second is ignored for the manager role, as in the
reference); optional flags select the model and the knobs of
``FederationConfig``.
"""
from __future__ import annotations

import argparse
import logging
import random
import sys
from typing import Optional

import torch
from aiohttp import web

from .config import FederationConfig
from .control import ExperimentWorker, Manager
from .data import linear_regression_shard
from .models import MLP2, LinearModel


def build_model(kind: str):
    if kind in ("lineartest", "linear"):
        return LinearModel()
    if kind == "mlp2":
        return MLP2()
    if kind == "resnet18":
        from .models import resnet18
        return resnet18(num_classes=10)
    if kind == "resnet50":
        from .models import resnet50
        return resnet50(num_classes=1000)
    if kind == "bert_base":
        from .models import bert_base
        return bert_base()
    raise SystemExit("unknown model {!r}".format(kind))


class LinearTestWorker(ExperimentWorker):
    """Example client with a fresh synthetic regression shard every round
    (reference demo.py:52-59)."""

    def __init__(self, *args, seed: Optional[int] = None, **kwargs):
        super().__init__(*args, **kwargs)
        self._rng = random.Random(seed)
        self._gen = torch.Generator()
        if seed is not None:
            self._gen.manual_seed(seed)

    def get_data(self):
        return linear_regression_shard(rng=self._rng, generator=self._gen)


def make_gpu_worker(app, model, host: str, port: int, cfg: FederationConfig):
    """One GPU-seated client (launch one per GPU under torchrun: RANK / LOCAL_RANK / WORLD_SIZE /
    MASTER_* come from the environment; NCCL only bootstraps the symmetric-memory rendezvous)."""
    import os

    import torch.distributed as dist

    from .control.gpu_worker import GpuExperimentWorker
    from .data import dirichlet_label_shards, image_shard, iid_label_shards
    rank, world = int(os.environ.get("RANK", "0")), int(os.environ.get("WORLD_SIZE", "1"))
    dev = torch.device("cuda", int(os.environ.get("LOCAL_RANK", "0")))
    torch.cuda.set_device(dev)
    if world > 1 and not dist.is_initialized():
        dist.init_process_group("nccl", device_id=dev)
    specs = (dirichlet_label_shards(world, cfg.num_classes, cfg.samples_per_client, cfg.alpha, cfg.seed)
             if cfg.partition == "dirichlet" else iid_label_shards(world, cfg.num_classes, cfg.samples_per_client))
    X, y = image_shard(specs[rank], seed=cfg.seed, dtype=torch.bfloat16, pin=True)
    return GpuExperimentWorker(app, model, host, device=dev, shard_fn=lambda: (X, y), backend=cfg.backend,
                               wire_dtype=cfg.wire_dtype, momentum=cfg.momentum, port=port,
                               heartbeat_time=cfg.heartbeat_time,
                               train_kwargs=cfg.train_kwargs())


def make_app(role: str, host: str, port: int, cfg: Optional[FederationConfig] = None) -> web.Application:
    cfg = cfg or FederationConfig()
    app = web.Application(client_max_size=1 << 34)
    model = build_model(cfg.model)
    if role == "manager":
        manager = Manager(app)
        manager.register_experiment(
            model, client_ttl=cfg.client_ttl, sample_k=cfg.sample_k, seed=cfg.seed, dataplane=cfg.backend,
            round_timeout=cfg.round_timeout, checkpoint_dir=cfg.checkpoint_dir,
            resume=bool(cfg.checkpoint_dir), dp=cfg.dp_config(), dp_delta=cfg.dp_delta, robust=cfg.robust_config())
        app["manager"] = manager
    elif role == "worker" and cfg.backend in ("fused", "nccl"):
        app["worker"] = make_gpu_worker(app, model, host, port, cfg)
    elif role == "worker":
        worker = LinearTestWorker(
            app, model, host, port=port, heartbeat_time=cfg.heartbeat_time,
            train_kwargs=cfg.train_kwargs(),
            seed=(cfg.seed * 1000 + port) if cfg.seed else None)
        app["worker"] = worker
    else:
        raise SystemExit("role must be 'manager' or 'worker'")
    return app


def main(argv=None) -> None:
    parser = argparse.ArgumentParser(description="baton_b200 demo (reference-compatible CLI)")
    parser.add_argument("role", choices=["manager", "worker"])
    parser.add_argument("host", help="manager address host:port (ignored for the manager role)")
    parser.add_argument("port", type=int, help="port to listen on")
    parser.add_argument("--bind", default=None, help="listen address (default: all interfaces)")
    parser.add_argument("-v", "--verbose", action="store_true")
    FederationConfig.add_arguments(parser)
    ns = parser.parse_args(argv)
    logging.basicConfig(level=logging.INFO if ns.verbose else logging.WARNING,
                        format="%(asctime)s %(name)s %(message)s")
    try:
        cfg = FederationConfig.from_args(ns)
    except ValueError as exc:
        parser.error(str(exc))
    app = make_app(ns.role, ns.host, ns.port, cfg)
    web.run_app(app, host=ns.bind, port=ns.port, print=print if ns.verbose else None)


if __name__ == "__main__":
    main(sys.argv[1:])
