"""SPMD federated engine: one process per GPU, every rank is a federated client.

This is the in-process counterpart of the HTTP control plane for jobs launched
with ``torchrun`` on one NVSwitch box (the ResNet / BERT benchmark configurations).
A *round* on every rank is

    (host -> device copy of this round's private shard, from pinned memory)
    local SGD for ``n_epoch`` epochs        (reference worker.py:103-106, demo.py:29-49)
    fused weighted reduce + broadcast + apply over NVLink   (manager.py:113-126 + :77-86)
    (device -> host read of the per-epoch losses)

with no host-side exchange between ranks: the sample counts n_k travel on the
collective's barrier flags.  Client sampling / logical clients stay in Python
(client sampling and round bookkeeping are host logic): with
``logical_clients > world`` each rank time-slices several logical clients and
folds their sample-weighted deltas locally before the cross-GPU reduce; the
per-round draw is a seeded ``random.Random`` shared by all ranks, so no
communication is needed to agree on the participants.
"""
from __future__ import annotations

import random
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Tuple

import torch

from ..metrics import phase
from ..train import GraphedLocalSGD, PortableLocalSGD, check_adamw, check_optimizer, check_prox_mu
from .arena import ParamArena
from .dp import DPConfig, RDPAccountant, check_dp, clip_factor
from .fedavg import FedAvgSession, NcclSession
from .robust import RobustConfig, check_aggregator, check_participants
from .scaffold import ScaffoldState


@dataclass
class RoundResult:
    update_name: str
    n_samples: int
    loss_history: List[float]
    participants: List[int] = field(default_factory=list)
    global_loss: Optional[List[float]] = None


@dataclass
class EvalResult:
    """Sample-weighted loss and accuracy of the global model on held-out data: ``loss`` / ``accuracy`` / ``n_samples``
    over every rank's shards, ``local_*`` over this rank's.  ``loss`` is the mean per-sample cross-entropy (or mean
    squared error); ``accuracy`` is 0 for regression; both are ``nan`` when no sample was evaluated."""
    loss: float
    accuracy: float
    n_samples: int
    local_loss: float
    local_accuracy: float
    local_n_samples: int


def _mean(total: float, n: float) -> float:
    return total / n if n > 0 else float("nan")


class FederatedEngine:
    def __init__(self, model, device, *, backend: str = "fused", group=None, loss: str = "ce",
                 lr: float = 0.05, batch_size: int = 128, momentum: float = 0.0, weight_decay: float = 0.0,
                 wire_dtype: str = "bf16", mode: str = "delta", n_ctas: Optional[int] = None, use_graph: bool = True,
                 logical_clients: int = 0, sample_k: Optional[int] = None, seed: int = 0, name: str = "exp",
                 nvls: "bool | str" = "auto", tile_flags: bool = False, prox_mu: float = 0.0,
                 dp_clip: float = 0.0, dp_noise_multiplier: float = 0.0, dp_seed: Optional[int] = None,
                 scaffold: bool = False, optimizer: str = "sgd", betas: Tuple[float, float] = (0.9, 0.999),
                 eps: float = 1e-8, aggregator: str = "mean", trim_ratio: float = 0.1):
        """``prox_mu > 0``: FedProx local training -- every step adds ``prox_mu * (theta - global_w)`` to the gradient,
        ``global_w`` being the global model the round started from (for logical clients too: each starts from it).

        ``dp_clip > 0``: DP-FedAvg (``parallel/dp.py``) -- every participating client's update is clipped to L2 norm
        ``dp_clip``, the participants are averaged uniformly and Gaussian noise of std ``dp_noise_multiplier * dp_clip``
        is added to the sum.  ``dp_seed``: Philox key of the noise (``None``: a secret random key; an explicit seed makes
        the noise predictable -- tests and reproductions only).  ``dp_clip = 0`` runs exactly the plain engine.

        ``scaffold=True``: SCAFFOLD (``parallel/scaffold.py``) -- every local step adds the correction ``c - c_i`` to
        the gradient, and each round also updates the control variates (option II), the server's one through the
        round's collective.  The model update stays the sample-weighted FedAvg mean.  :meth:`control_variates` reads
        them.  It cannot be combined with DP, FedProx, ``mode='weights'`` or ``tile_flags``.

        ``optimizer="adamw"``: every client's local steps are those of a fresh ``torch.optim.AdamW(lr, betas, eps,
        weight_decay)`` (one parameter group, weight decay on every parameter), created anew for each client and
        round; the server update stays the FedAvg mean.  It cannot be combined with ``momentum``, SCAFFOLD or FedProx.
        The second moment costs one more fp32 buffer over the parameters.

        ``aggregator="median"`` / ``"trimmed_mean"`` (``parallel/robust.py``): the round's update is the coordinate-wise
        median or ``trim_ratio``-trimmed mean of the participating clients' deltas, unweighted, instead of the
        sample-weighted mean (``"mean"``, the default, runs exactly the plain engine).  At most 32 participants per
        round.  Every hosted participant uploads its own wire segment instead of being folded: ``S = min(ceil(L /
        world), sample_k or L)`` segments for ``L`` logical clients, which costs ``2 * S * wire bytes`` of symmetric
        memory per GPU (16 segments of a bf16 ResNet-18 are about 0.7 GB).  It cannot be combined with DP, SCAFFOLD,
        ``mode='weights'`` or ``tile_flags``; FedProx, AdamW, momentum and the fp8 wire combine freely."""
        prox_mu = check_prox_mu(prox_mu)
        adam = check_optimizer(optimizer, momentum, prox_mu=prox_mu)
        if adam:
            if scaffold:
                raise ValueError("AdamW with SCAFFOLD is not supported: option II's dc = (x - theta) / (K lr) - c "
                                 "assumes SGD steps")
            betas, eps = check_adamw(betas, eps)
        dp_clip, dp_noise_multiplier = check_dp(dp_clip, dp_noise_multiplier)
        if scaffold:
            if dp_clip > 0.0:
                raise ValueError("SCAFFOLD with DP-FedAvg is not supported: DP would also have to clip and noise dc")
            if prox_mu > 0.0:
                raise ValueError("SCAFFOLD and FedProx (prox_mu > 0) are exclusive")
            if mode != "delta":
                raise ValueError("SCAFFOLD needs mode='delta'")
            if tile_flags:
                raise ValueError("SCAFFOLD with tile_flags is not supported: the correction c - c_i reads c, which "
                                 "the previous round's collective writes, so it cannot run ahead of the join")
        trim_ratio = check_aggregator(aggregator, trim_ratio)
        self.robust = RobustConfig(aggregator, trim_ratio) if aggregator != "mean" else None
        if self.robust is not None:
            if dp_clip > 0.0:
                raise ValueError("a robust aggregator with DP-FedAvg is not supported: DP's noise is calibrated to the "
                                 "clipped mean")
            if scaffold:
                raise ValueError("a robust aggregator with SCAFFOLD is not supported: its control-variate update is a "
                                 "mean")
            if mode != "delta":
                raise ValueError("a robust aggregator needs mode='delta'")
            if tile_flags:
                raise ValueError("a robust aggregator with tile_flags is not supported")
        self.dp = DPConfig(dp_clip, dp_noise_multiplier, dp_seed) if dp_clip > 0.0 else None
        if self.dp is not None and mode != "delta":
            raise ValueError("DP-FedAvg needs mode='delta'")
        self.device = torch.device(device)
        self.model = model
        self.name = name
        self.arena = ParamArena(model, self.device, momentum=momentum > 0)
        if hasattr(model, "build_workspace"):
            model.build_workspace(self.device)
        if self.device.type == "cuda":
            self.trainer = GraphedLocalSGD(model, self.arena, loss=loss, use_graph=use_graph)
            model._graphed_trainer = self.trainer
        else:
            # CPU / gloo: the plumbing configuration -- same engine, portable PyTorch training loop, and the
            # torch.distributed session (the fused collective needs NVLink peer memory)
            if backend == "fused":
                raise ValueError("backend='fused' needs CUDA devices; use backend='nccl' (torch.distributed, "
                                 "gloo on CPU) for CPU runs")
            self.trainer = PortableLocalSGD(model, self.arena, loss=loss)
        Session = {"fused": FedAvgSession, "nccl": NcclSession}[backend]
        robust_kw = {}
        if self.robust is not None:
            world = self._group_size(group)
            population = logical_clients if logical_clients and logical_clients > world else world
            check_participants(min(sample_k, population) if sample_k else population)
            per_rank = -(-population // world) if population > world else 1
            robust_kw = {"robust": self.robust, "max_clients": min(per_rank, sample_k or population)}
        self.session = Session(self.arena, group, wire_dtype=wire_dtype, mode=mode, n_ctas=n_ctas, nvls=nvls,
                               tile_flags=tile_flags, dp=self.dp, scaffold=scaffold, **robust_kw)
        self.dp = self.session.dp                  # rank 0's noise key
        self.accountant = RDPAccountant(self.dp.noise_multiplier) if self.dp is not None else None
        self.backend = backend
        self.rank, self.world = self.session.rank, self.session.world
        # K4: the last SGD step of the captured epoch writes the upload copy itself (no pack phase in the collective);
        # only for the plain one-client-per-GPU rounds -- logical clients fold their deltas after training
        self.prepack = (backend == "fused" and self.device.type == "cuda"
                        and not (logical_clients and logical_clients > self.world))
        if self.prepack and hasattr(self.session, "pack_spec"):
            self.trainer.pack = self.session.pack_spec()
        # the round-end collective runs on the session's high-priority side stream: the NEXT round's host->device shard
        # copy (and anything else that does not touch the arena) overlaps it; local training joins first
        self.overlap_collective = backend == "fused" and self.device.type == "cuda"
        # K3 (bcast_gemm) on the flagship path: the first convolution's weight staging + GEMM acquire the collective's
        # arrival flags, and the head of the next round's captured epoch runs while the collective is still in flight
        self.k3 = bool(self.overlap_collective and tile_flags and hasattr(model, "conv1")
                       and isinstance(self.session, FedAvgSession) and hasattr(self.session, "gate_first_conv")
                       and hasattr(self.trainer, "k3_join"))
        if self.k3:
            self.session.gate_first_conv(model.conv1)
            self.trainer.k3_join = self.sync
        self.hp = dict(lr=lr, batch_size=batch_size, momentum=momentum, weight_decay=weight_decay, prox_mu=prox_mu)
        if adam:
            self.hp.update(optimizer=optimizer, betas=betas, eps=eps)
        self.n_rounds = 0
        self.logical_clients = logical_clients if logical_clients and logical_clients > self.world else 0
        self.sample_k = sample_k
        self.scaf = ScaffoldState(self.arena.n_param, self.device) if scaffold else None
        self._rng = random.Random(seed)            # identical stream on every rank
        self._stage: Dict[Tuple, Tuple[torch.Tensor, torch.Tensor]] = {}
        self._eval_stage: Dict[Tuple, Tuple[torch.Tensor, torch.Tensor]] = {}
        self._acc = None
        self._dp_rec = None              # DP with logical clients: [clip factor, norm] per hosted client of the round
        self._dp_n = 0
        self._dp_work = None             # ... the norm kernel's partials (CUDA)
        self._dp_bad = 0                 # ... non-finite client updates so far (device counter on CUDA)
        self.last_losses_dev = None
        self.samples_trained = 0          # samples this rank pushed through local SGD (per epoch)
        self.phase_s: Dict[str, float] = {}   # host seconds per NVTX phase (launch cost; device time is in bench.py)

    @staticmethod
    def _group_size(group) -> int:
        import torch.distributed as dist
        return dist.get_world_size(group) if dist.is_available() and dist.is_initialized() else 1

    # ------------------------------------------------------------------ data staging
    def stage(self, X_host: torch.Tensor, y_host: torch.Tensor, slot: int = 0):
        """Asynchronous host->device copy of a shard into persistent staging buffers (so the
        captured epoch graph keeps pointing at the same addresses).  ``X_host``/``y_host`` should
        be pinned.  Returns the device views."""
        return self._copy_in(self._stage, X_host, y_host, slot)

    def _copy_in(self, stage: dict, X_host: torch.Tensor, y_host: torch.Tensor, slot: int):
        key = (slot, tuple(X_host.shape), X_host.dtype, tuple(y_host.shape), y_host.dtype)
        bufs = stage.get(key)
        if bufs is None:
            bufs = (torch.empty(X_host.shape, dtype=X_host.dtype, device=self.device),
                    torch.empty(y_host.shape, dtype=y_host.dtype, device=self.device))
            stage[key] = bufs
        bufs[0].copy_(X_host, non_blocking=True)
        bufs[1].copy_(y_host, non_blocking=True)
        return bufs

    @staticmethod
    def h2d_bytes(X_host: torch.Tensor, y_host: torch.Tensor) -> int:
        return X_host.numel() * X_host.element_size() + y_host.numel() * y_host.element_size()

    # ------------------------------------------------------------------ participants
    def draw_participants(self) -> List[int]:
        """Logical client ids taking part in this round (same on every rank)."""
        total = self.logical_clients or self.world
        ids = list(range(total))
        if self.sample_k is None or self.sample_k >= total:
            return ids
        return sorted(self._rng.sample(ids, self.sample_k))

    def hosted(self, client_id: int) -> bool:
        return client_id % self.world == self.rank

    # ------------------------------------------------------------------ one round
    def run_round(self, shards, n_epoch: int = 1, read_loss: bool = True) -> RoundResult:
        """``shards``: for a plain run a ``(X, y)`` pair (device tensors, or pinned host tensors
        that are staged first); with logical clients a callable ``client_id -> (X, y)``."""
        update_name = "update_{}_{:05d}".format(self.name, self.n_rounds)
        participants = self.draw_participants()
        mine = [c for c in participants if self.hosted(c)]
        a = self.arena
        total_n = 0
        losses_dev = None
        if not self.logical_clients:
            if mine:
                X, y = shards(self.rank) if callable(shards) else shards
                if not X.is_cuda:
                    with phase("baton.h2d_shard", self.phase_s):
                        X, y = self.stage(X, y)
                if not self.k3:
                    self.sync()              # the previous round's collective must have landed before training reads theta
                if self.prepack and self.trainer.pack is not None:
                    self.session.arm_prepack(float(X.shape[0]))
                with phase("baton.local_train", self.phase_s):
                    losses_dev = self._train_client(self.rank, X, y, n_epoch, first=True)
                total_n = X.shape[0]
        elif self.robust is not None:
            # robust: every hosted participant uploads its own segment (a median of per-rank sums is not a median of
            # clients); the next co-resident client starts from the global model
            self.sync()
            for j, cid in enumerate(mine):
                X, y = shards(cid)
                if not X.is_cuda:
                    X, y = self.stage(X, y, slot=j)
                ld = self._train_client(cid, X, y, n_epoch, first=(j == 0))
                nk = X.shape[0]
                losses_dev = ld * nk if losses_dev is None else losses_dev + ld * nk
                total_n += nk
                self.session.pack_client(j, reset=j + 1 < len(mine))
            if losses_dev is not None and total_n:
                losses_dev = losses_dev / total_n
        else:
            # time-sliced logical clients: fold n_k * (theta_k - global) locally, then upload the mean
            # (DP: s_k * (theta_k - global) for every hosted client, even a single one, and the mean over clients)
            self.sync()
            fold = len(mine) > 1 or (self.dp is not None and mine)
            if fold and self._acc is None:
                self._acc = torch.zeros_like(a.theta)
            if fold and not a.theta.is_cuda:
                self._acc.zero_()
            if self.dp is not None:
                self._dp_begin(len(mine))
            for j, cid in enumerate(mine):
                X, y = shards(cid)
                if not X.is_cuda:
                    X, y = self.stage(X, y, slot=j)
                ld = self._train_client(cid, X, y, n_epoch, first=(j == 0))
                nk = X.shape[0]
                losses_dev = ld * nk if losses_dev is None else losses_dev + ld * nk
                total_n += nk
                if self.dp is not None:
                    self._dp_fold(j, more=j + 1 < len(mine))
                elif len(mine) > 1:
                    more = j + 1 < len(mine)           # the next co-resident client starts from the global model
                    if a.theta.is_cuda:
                        from ..ops import functional as F     # ONE kernel: fold the delta + reset the replica
                        F.fold_client(self._acc, a.theta, a.global_w, nk, first=(j == 0), reset=more,
                                      w_bf16=a.theta_bf16, momentum=a.momentum)
                    else:
                        self._acc.add_(a.theta - a.global_w, alpha=float(nk))
                        if more:
                            a.theta.copy_(a.global_w)
                            a.sync_shadow()
                            if a.momentum is not None:
                                a.momentum.zero_()
            if fold:
                m_r = len(mine) if self.dp is not None else total_n
                if a.theta.is_cuda:
                    from ..ops import functional as F
                    F.fold_finish(self._acc, a.theta, a.global_w, m_r)
                else:
                    torch.add(a.global_w, self._acc, alpha=1.0 / m_r, out=a.theta)
            if losses_dev is not None and total_n:
                losses_dev = losses_dev / total_n
        self.last_losses_dev = losses_dev
        self.samples_trained += int(total_n)
        loss_for_wire = None
        if losses_dev is not None:
            steps = max(1, self.trainer.last_steps)
            loss_for_wire = losses_dev[:, 0] / steps
        # DP: the weights count clients (1 per seat, m_r with logical clients), not samples
        my_n = float(total_n) if self.dp is None else float(len(mine) if self.logical_clients else (1 if mine else 0))
        with phase("baton.aggregate_broadcast", self.phase_s):
            self._aggregate(my_n, loss_for_wire, clipped=bool(self.dp is not None and self.logical_clients),
                            n_clients=len(mine) if (self.robust is not None and self.logical_clients) else None)
        if self.accountant is not None:
            self.accountant.step(len(participants) / float(self.logical_clients or self.world))
        self.n_rounds += 1
        hist: List[float] = []
        if read_loss and losses_dev is not None:
            hist = loss_for_wire.tolist()       # device -> host read of the round's result
        return RoundResult(update_name, int(total_n), hist, participants)

    def _train_client(self, cid: int, X, y, n_epoch: int, first: bool):
        """Local training of client ``cid`` on the replica; with SCAFFOLD, its correction before and its control-variate
        update after (before any fold resets the replica)."""
        if self.scaf is None:
            return self.trainer.run(X, y, n_epoch=n_epoch, return_device=True, **self.hp)
        self.scaf.begin_client(cid)
        ld = self.trainer.run(X, y, n_epoch=n_epoch, return_device=True, corr=self.scaf.corr, **self.hp)
        self.scaf.end_client(cid, self.arena, n_epoch * self.trainer.last_steps, self.hp["lr"], first=first)
        return ld

    def control_variates(self):
        """SCAFFOLD's ``(c, {client_id: c_i})``: the server control variate and those of the clients this rank hosts
        that have taken part so far (fp32 tensors over the parameters, on the engine's device; live, not copies)."""
        if self.scaf is None:
            raise RuntimeError("SCAFFOLD is off (scaffold=False)")
        self.sync()
        return self.scaf.c, dict(self.scaf.c_i)

    def sync(self) -> None:
        """Make the compute stream wait for a collective that is still running on the side stream (call before
        anything reads or writes the arena: training, ``state_dict()``, checkpoints)."""
        join = getattr(self.session, "join", None)
        if join is not None:
            join()

    # ------------------------------------------------------------------ differential privacy
    def _dp_begin(self, n_mine: int) -> None:
        dev = self.arena.theta.device
        if self._dp_rec is None or self._dp_rec.shape[0] < max(n_mine, 1):
            self._dp_rec = torch.zeros(max(n_mine, 1), 2, dtype=torch.float32, device=dev)
        if self._dp_work is None and dev.type == "cuda":
            from ..ops._ext import load
            self._dp_work = torch.zeros(load().DP_WORK_WORDS, dtype=torch.int64, device=dev)
            self._dp_bad = torch.zeros(1, dtype=torch.int32, device=dev)
        self._dp_n = n_mine

    def _dp_fold(self, j: int, more: bool) -> None:
        """Clip hosted client ``j``'s update into the accumulator and (``more``) reset the replica for the next one.
        On CUDA the factor stays on the device: norm kernel -> device scalar -> scaled fold, no host synchronisation."""
        a = self.arena
        if a.theta.is_cuda:
            from ..ops import functional as F
            rec = self._dp_rec[j]
            F.dp_clip_factor(a.theta, a.global_w, self.dp.clip, self._dp_work, rec[0:1], rec[1:2], nonfinite=self._dp_bad)
            F.fold_client_scaled(self._acc, a.theta, a.global_w, rec[0:1], first=(j == 0), reset=more,
                                 w_bf16=a.theta_bf16, momentum=a.momentum)
            return
        sj, norm = clip_factor(a.theta - a.global_w, self.dp.clip)
        self._dp_rec[j, 0], self._dp_rec[j, 1] = sj, norm
        if sj == 0.0:
            self._dp_bad += 1
        else:
            self._acc.add_(a.theta - a.global_w, alpha=sj)
        if more:
            a.theta.copy_(a.global_w)
            a.sync_shadow()
            if a.momentum is not None:
                a.momentum.zero_()

    def last_clip_factors(self) -> List[float]:
        """Clip factors ``s`` of the clients this rank trained in the last round (a host read)."""
        if self.dp is None:
            return []
        self.sync()
        if self.logical_clients:
            return self._dp_rec[: self._dp_n, 0].tolist() if self._dp_rec is not None else []
        return self.session.last_clip_factors()

    def last_update_norms(self) -> List[float]:
        """L2 norms of the updates of the clients this rank hosted in the last logical-client DP round (a host read)."""
        if self.dp is None or not self.logical_clients or self._dp_rec is None:
            return []
        self.sync()
        return self._dp_rec[: self._dp_n, 1].tolist()

    def nonfinite_updates(self) -> int:
        """Client updates of this rank so far whose norm was not finite (clipped to nothing, still counted in m)."""
        if self.dp is None:
            return 0
        self.sync()
        return int(self._dp_bad) + self.session.nonfinite_updates()

    def privacy_spent(self, delta: float = 1e-5):
        """``(epsilon, order)`` of the DP rounds run so far at ``delta`` (RDP accountant of the sampled Gaussian
        mechanism; a fixed-size participant sample is accounted as Poisson sampling at rate k / K)."""
        if self.accountant is None:
            raise RuntimeError("differential privacy is off (dp_clip = 0)")
        return self.accountant.get_privacy_spent(delta)

    def _aggregate(self, my_n: float, loss_dev, clipped: bool = False, n_clients: Optional[int] = None) -> None:
        s = self.session
        if self.robust is not None:    # n_clients: segments packed by pack_client (logical clients), else seg 0 as usual
            kw = self._aggregate_kwargs(s, my_n, loss_dev)
            if n_clients is not None:
                kw["n_clients"] = n_clients
            s.aggregate(my_n=my_n, **kw)
            return
        if self.scaf is not None:      # SCAFFOLD: c += (sum of the ranks' dc) / N in the same collective
            s.aggregate(my_n=my_n, control=(self.scaf.c, self.scaf.up, self.logical_clients or self.world),
                        **self._aggregate_kwargs(s, my_n, loss_dev))
            return
        if self.dp is not None:
            kw = {"clipped": clipped}
            if isinstance(s, FedAvgSession):
                kw["on_side_stream"] = bool(self.overlap_collective)
                kw["prepacked"] = bool(self.prepack and getattr(self.trainer, "emitted_wire", False) and my_n > 0
                                       and not getattr(self.trainer, "last_had_tail_step", False))
            if loss_dev is not None and hasattr(s, "loss_local"):
                k = min(loss_dev.numel(), s.loss_local.numel())
                s.loss_local.zero_()
                s.loss_local[:k].copy_(loss_dev[:k])
                s.aggregate(my_n=my_n, **kw)
            else:
                s.aggregate(my_n=my_n, loss_history=loss_dev.tolist() if loss_dev is not None else None, **kw)
            return
        side = bool(self.overlap_collective and isinstance(s, FedAvgSession))
        if loss_dev is not None and hasattr(s, "loss_local"):
            k = min(loss_dev.numel(), s.loss_local.numel())
            s.loss_local.zero_()
            s.loss_local[:k].copy_(loss_dev[:k])
            pre = bool(self.prepack and getattr(self.trainer, "emitted_wire", False) and my_n > 0
                       and not getattr(self.trainer, "last_had_tail_step", False))
            s.aggregate(my_n=my_n, prepacked=pre, on_side_stream=side) if isinstance(s, FedAvgSession) else s.aggregate(my_n=my_n)
        elif loss_dev is not None:
            s.aggregate(my_n=my_n, loss_history=loss_dev.tolist())
        else:
            s.aggregate(my_n=my_n)

    def _aggregate_kwargs(self, s, my_n: float, loss_dev) -> dict:
        """Loss, upload and stream arguments of a round's ``aggregate`` (the plain round's choices)."""
        kw = {}
        if isinstance(s, FedAvgSession):
            kw["on_side_stream"] = bool(self.overlap_collective)
            kw["prepacked"] = bool(self.prepack and getattr(self.trainer, "emitted_wire", False) and my_n > 0
                                   and not getattr(self.trainer, "last_had_tail_step", False))
        if loss_dev is not None and hasattr(s, "loss_local"):
            k = min(loss_dev.numel(), s.loss_local.numel())
            s.loss_local.zero_()
            s.loss_local[:k].copy_(loss_dev[:k])
        elif loss_dev is not None:
            kw["loss_history"] = loss_dev.tolist()
        return kw

    def global_loss(self, n_epoch: int) -> List[float]:
        return self.session.reduced_loss(n_epoch)

    # ------------------------------------------------------------------ evaluation
    def evaluate(self, shards, batch_size: Optional[int] = None) -> EvalResult:
        """Loss and accuracy of the global model on held-out data.  ``shards`` takes the forms of :meth:`run_round`:
        an ``(X, y)`` pair for this rank, a callable ``rank -> (X, y)``, or with logical clients a callable
        ``client_id -> (X, y)`` (every client this rank hosts is evaluated and the results are summed); ``None`` or
        an empty shard contributes nothing.  Host shards are staged into their own buffers, never the training ones.
        Nothing of the model, the arena or the training state changes.  Every rank must call it: the global numbers
        come from one all-reduce of ``[loss sum, #correct, n]`` over the session's process group."""
        self.sync()          # the round-end collective may still be writing the arena on its side stream
        batch = int(batch_size or self.hp["batch_size"])
        if self.logical_clients:
            ids = [c for c in range(self.logical_clients) if self.hosted(c)]
            pairs = [shards(c) for c in ids] if shards is not None else []
        elif shards is None:
            pairs = []
        else:
            pairs = [shards(self.rank) if callable(shards) else shards]
        loss = correct = n = 0.0
        for pair in pairs:
            if pair is None or pair[0].shape[0] == 0:
                continue
            X, y = pair
            if self.device.type == "cuda" and not X.is_cuda:
                # one staging buffer per shape: a pass ends with a host read, so the next shard may overwrite it
                X, y = self._copy_in(self._eval_stage, X, y, 0)
            ls, c, k = self.trainer.evaluate(X, y, batch_size=batch)
            loss, correct, n = loss + ls, correct + c, n + k
        tot = [loss, correct, n]
        group = getattr(self.session, "group", None)
        if self.world > 1 and torch.distributed.is_available() and torch.distributed.is_initialized():
            t = torch.tensor(tot, dtype=torch.float64, device=self.device)
            torch.distributed.all_reduce(t, group=group)
            tot = t.tolist()
        return EvalResult(loss=_mean(tot[0], tot[2]), accuracy=_mean(tot[1], tot[2]), n_samples=int(tot[2]),
                          local_loss=_mean(loss, n), local_accuracy=_mean(correct, n), local_n_samples=int(n))

    def state_dict(self):
        self.sync()
        return self.model.state_dict()
