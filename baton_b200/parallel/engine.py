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
from typing import Dict, List, Optional, Sequence, Tuple

import torch

from ..metrics import phase
from ..train import GraphedLocalSGD, PortableLocalSGD, check_adamw, check_max_grad_norm, check_prox_mu
from .arena import ParamArena
from .compress import TopKConfig, TopKState
from .dp import DPConfig, RDPAccountant, check_dp, clip_factor
from .features import check_features, round_plan
from .fedavg import FedAvgSession, NcclSession
from .personal import LocalStore, resolve_local_keys
from .robust import RobustConfig, check_aggregator, check_krum_participants, check_participants
from .server_opt import ServerOptConfig
from .scaffold import ScaffoldState
from .secagg import SecAggConfig


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
                 eps: float = 1e-8, aggregator: str = "mean", trim_ratio: float = 0.1, krum_f: int = 0,
                 krum_m: Optional[int] = None, server_opt: Optional[str] = None, server_lr: Optional[float] = None,
                 server_betas: Tuple[float, float] = (0.9, 0.99), server_tau: float = 1e-3,
                 compress: Optional[str] = None, topk_ratio: float = 0.01, error_feedback: bool = True,
                 local_keys: "Optional[str | Sequence[str]]" = None, augment: Optional[str] = None,
                 augment_padding: int = 4, mix: Optional[str] = None, mix_alpha: float = 1.0,
                 label_smoothing: float = 0.0, max_grad_norm: float = 0.0, secure_agg: bool = False,
                 secagg_range: float = 64.0):
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
        ``mode='weights'`` or ``tile_flags``; FedProx, AdamW, momentum and the fp8 wire combine freely.

        ``aggregator="krum"``: Multi-Krum -- each participant is scored by its summed squared distances to its nearest
        ``P - krum_f - 2`` fellow participants, and the plain mean of the ``krum_m`` best-scoring updates (default ``P -
        krum_f``; 1 is classic Krum) is applied.  The planned participants per round must number at least ``2 krum_f +
        3``; a round with fewer still runs, with ``k`` and ``m`` clamped (``parallel/robust.py``).  The other robust
        aggregators' rules and costs apply.  :meth:`last_krum` reports the last round's scores by client id.

        ``server_opt="avgm"`` / ``"adagrad"`` / ``"yogi"`` / ``"adam"`` (``parallel/server_opt.py``): FedAvgM, FedAdagrad,
        FedYogi or FedAdam on the server -- the round's aggregate, whichever aggregator computed it, drives a stateful
        step of size ``server_lr`` (required) with ``server_betas`` and ``server_tau`` on the parameters; buffers keep
        ``global += aggregate``.  The state costs one (FedAvgM) or two fp32 buffers over the parameters on every rank;
        :meth:`server_state` reads it.  It needs ``mode='delta'``.  ``None`` (the default) runs exactly the plain
        engine.

        ``compress="topk"`` (``parallel/compress.py``): every participating client uploads only its ``k = max(1,
        ceil(topk_ratio * n_float))`` largest-magnitude update entries (``n_float``: the float ``state_dict`` elements);
        with ``error_feedback`` the rest is carried in a per-client fp32 residual over the arena, kept on the rank that
        hosts the client (:meth:`topk_residuals`), and added to its next update.  The round's update is the
        sample-weighted mean of the sparse uploads; the downlink stays dense.  It cannot be combined with the fp8 wire,
        DP, a robust aggregator, SCAFFOLD, ``mode='weights'`` or ``tile_flags``; FedProx, AdamW, momentum, logical
        clients and every server optimizer combine freely.  :meth:`last_upload_bytes` reports the upload.  ``None``
        (the default) runs exactly the plain engine.

        ``local_keys`` (``parallel/personal.py``): personalized FL -- the named float ``state_dict`` entries stay with
        each client and out of the collective: ``"bn"`` (FedBN: every BatchNorm's weight, bias and running statistics),
        ``"head"`` (FedPer: the model's ``head`` entries), ``state_dict`` keys or ``fnmatch`` patterns, or a sequence
        mixing them.  Every client (logical clients included) starts from the model's values at construction the first
        time it trains and keeps what its last training left; FedProx's anchor for a local entry is the client's own
        value.  The shared entries follow the plain round (with a server optimizer if one is set); integer buffers stay
        shared.  :meth:`client_state_dict` and :meth:`local_entries` read a hosted client's model and entries,
        :meth:`evaluate` scores each hosted client's personalized model, and :meth:`state_dict` returns the local
        entries at their initial values.  It cannot be combined with DP, SCAFFOLD, a robust aggregator or Krum, top-k
        uploads or ``tile_flags``; the optimizer-emitted upload is off.  Each hosted client that has taken part costs
        ``4 (hi - lo)`` bytes.  ``None`` (the default) runs exactly the plain engine.

        ``augment="crop"`` / ``"flip"`` / ``"crop_flip"`` (``data/augment.py``): every client's local epochs train on
        random crops of the zero-padded images (``augment_padding`` pixels each side) and random horizontal flips,
        drawn afresh per sample and epoch inside the batch gather.  The key is derived from ``seed`` (the same on every
        rank) and each client's stream is ``(round_index << 32) | client_id``, so co-hosted clients and successive
        rounds draw independently and a run is reproducible from its seed.  Shards must be NHWC images.  It is local to
        each client and combines with every other option.  ``None`` (the default) runs exactly the plain engine.

        ``mix="mixup"`` / ``"cutmix"`` / ``"mixup_cutmix"`` (with ``mix_alpha``) and ``label_smoothing``
        (``data/mix.py``): every client trains on batches mixed with themselves rolled by one, one lambda per batch, and
        on the soft-target cross-entropy.  Mixing draws from the augmentation key and the client's stream of the round,
        with or without ``augment``.  It needs the cross-entropy loss, and mixing needs NHWC image shards; both are
        local to each client and combine with every other option.  Evaluation keeps hard labels.  ``None`` / ``0``
        (the defaults) run exactly the plain engine.

        ``max_grad_norm > 0``: every local step clips the gradient of the loss to this 2-norm, as
        ``torch.nn.utils.clip_grad_norm_(model.parameters(), max_grad_norm)`` right after backward and before weight
        decay, FedProx, SCAFFOLD, momentum or AdamW act.  The norm covers every trained parameter, client-local ones
        included.  It is local to each client and combines with every other option; it is not DP (``dp_clip`` clips
        client updates).  :meth:`last_grad_norms` reports the pre-clip norms.  ``0`` (the default) runs exactly the
        plain engine.

        ``secure_agg=True`` (``parallel/secagg.py``): secure aggregation -- every rank clamps its update to
        ``[-secagg_range, secagg_range]``, encodes its weighted share in fixed point and uploads it under pairwise ChaCha20
        masks that cancel in the ring sum, so no rank's upload is readable in the clear through the symmetric mapping.
        The rank is the party: logical clients it hosts are folded before the upload and are not hidden from each
        other.  The counts, the losses and integer buffers are not masked.  It needs ``wire_dtype='fp32'`` and
        ``mode='delta'``; it cannot be combined with DP, a robust aggregator or Krum, top-k uploads, SCAFFOLD,
        client-local entries or ``tile_flags``; every server optimizer, FedProx, AdamW, momentum, augmentation, mixing,
        gradient clipping, logical clients and sampling combine.  The optimizer-emitted upload is off.
        :meth:`last_secagg_saturation` reports this rank's clamped elements.  ``False`` (the default) runs exactly the
        plain engine."""
        from ..data.augment import check_augment
        from ..data.mix import check_mix, check_mix_loss
        aug = check_augment(augment, augment_padding)
        mixc = check_mix(mix, mix_alpha, label_smoothing)
        check_mix_loss(mixc, loss)
        if compress not in (None, "topk"):
            raise ValueError("compress must be None or 'topk', got {!r}".format(compress))
        self.topk = TopKConfig(topk_ratio, error_feedback) if compress == "topk" else None
        sopt = None
        if server_opt is not None:
            b1, b2 = server_betas
            sopt = ServerOptConfig(server_opt, server_lr, b1, b2, server_tau)
        prox_mu = check_prox_mu(prox_mu)
        max_grad_norm = check_max_grad_norm(max_grad_norm)
        adam = optimizer == "adamw"
        if adam:
            betas, eps = check_adamw(betas, eps)
        dp_clip, dp_noise_multiplier = check_dp(dp_clip, dp_noise_multiplier)
        trim_ratio = check_aggregator(aggregator, trim_ratio)
        self.robust = RobustConfig(aggregator, trim_ratio, krum_f, krum_m) if aggregator != "mean" else None
        self.dp = DPConfig(dp_clip, dp_noise_multiplier, dp_seed) if dp_clip > 0.0 else None
        keys = resolve_local_keys(model, local_keys) if local_keys is not None else None
        if not isinstance(secure_agg, bool):
            raise TypeError("secure_agg must be a bool, got {!r}".format(secure_agg))
        self.secagg = SecAggConfig(secagg_range) if secure_agg else None
        check_features(wire_dtype=wire_dtype, mode=mode, dp=self.dp, scaffold=scaffold, robust=self.robust,
                       topk=self.topk, server_opt=sopt, tile_flags=tile_flags, optimizer=optimizer, momentum=momentum,
                       prox_mu=prox_mu, local=keys is not None, secure_agg=secure_agg,
                       frozen=any(not p.requires_grad for p in model.parameters()),
                       vit=getattr(model, "is_vit", False))
        self.device = torch.device(device)
        self.model = model
        self.name = name
        self.arena = ParamArena(model, self.device, momentum=momentum > 0, local=keys or ())
        self.personal = LocalStore(self.arena, keys) if keys is not None else None
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
        # robust: one segment per hosted client; top-k with logical clients: the folded upload is the union of their
        # supports
        max_clients = 1
        if self.robust is not None or self.topk is not None:
            planned, max_clients = round_plan(self._group_size(group), logical_clients, sample_k)
            if self.robust is not None:
                check_participants(planned)
                if self.robust.kind == "krum":
                    check_krum_participants(planned, self.robust.krum_f)
        self.session = Session(self.arena, group, wire_dtype=wire_dtype, mode=mode, n_ctas=n_ctas, nvls=nvls,
                               tile_flags=tile_flags, dp=self.dp, scaffold=scaffold, server_opt=sopt,
                               robust=self.robust, topk=self.topk, max_clients=max_clients,
                               local=self.personal is not None, secagg=self.secagg)
        if self.arena.frozen_range is not None:
            self._check_frozen_agree(group)
        self.dp = self.session.dp                  # rank 0's noise key
        self.accountant = RDPAccountant(self.dp.noise_multiplier) if self.dp is not None else None
        self.backend = backend
        self.rank, self.world = self.session.rank, self.session.world
        # K4: the last SGD step of the captured epoch writes the upload copy itself (no pack phase in the collective);
        # only for the plain one-client-per-GPU rounds -- logical clients fold their deltas after training
        self.prepack = (backend == "fused" and self.device.type == "cuda" and self.topk is None
                        and self.personal is None and self.secagg is None
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
        if max_grad_norm > 0:
            self.hp.update(max_grad_norm=max_grad_norm)
        self._grad_norms: Dict[int, torch.Tensor] = {}     # client id -> [n_epoch, steps] norms of the last round
        aug_hp = {}
        if aug is not None:
            aug_hp.update(augment=aug.kind, augment_padding=aug.padding)
        if mixc is not None:
            aug_hp.update(mix=mixc.kind, mix_alpha=mixc.alpha, label_smoothing=mixc.smoothing)
        # dropout (a BERT model with a nonzero probability) draws from the same key and per-client stream
        self.aug_hp = dict(aug_hp, augment_seed=seed) if aug_hp or getattr(model, "has_dropout", False) else None
        self.n_rounds = 0
        self._last_participants: Optional[List[int]] = None
        self.logical_clients = logical_clients if logical_clients and logical_clients > self.world else 0
        self.sample_k = sample_k
        self.scaf = ScaffoldState(self.arena.n_param, self.device) if scaffold else None
        self.topk_state = (TopKState(self.arena.n, self.device)
                           if self.topk is not None and self.topk.error_feedback else None)
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

    def _check_frozen_agree(self, group) -> None:
        """The collective never carries the frozen range, so every rank must start from the same frozen weights: one
        hash of the range, all-reduced as (max, -min), and a ``ValueError`` on every rank when they differ."""
        import hashlib
        import torch.distributed as dist
        if not (dist.is_available() and dist.is_initialized()) or self._group_size(group) == 1:
            return
        lo, hi = self.arena.frozen_range
        digest = hashlib.sha256(self.arena.theta[lo:hi].cpu().numpy().tobytes()).digest()
        h = int.from_bytes(digest[:7], "little")           # fits an int64 with its negation
        t = torch.tensor([h, -h], dtype=torch.int64, device=self.device)
        dist.all_reduce(t, op=dist.ReduceOp.MAX, group=group)
        if int(t[0]) != -int(t[1]):
            raise ValueError("the frozen parameters differ between ranks: every client must start from the same base "
                             "weights, which the collective never carries")

    def lora_state_dict(self) -> dict:
        """The model's adapter and classifier entries under Hugging-Face names (``models/bert.py``)."""
        self.sync()
        return self.model.lora_state_dict()

    def merged_hf_state_dict(self) -> dict:
        """A stock Hugging-Face ``state_dict`` with the adapters merged into the base weights (``models/bert.py``)."""
        self.sync()
        return self.model.merged_hf_state_dict()

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
        self._last_participants = participants
        self._grad_norms = {}
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
                if self.personal is not None:    # the replica holds its client's local entries across rounds
                    self.personal.refresh()
                with phase("baton.local_train", self.phase_s):
                    losses_dev = self._train_client(self.rank, X, y, n_epoch, first=True)
                if self.personal is not None:
                    self.personal.swap_out(self.rank)
                total_n = X.shape[0]
                if self.topk is not None:
                    self.session.pack_topk(self._residual(self.rank))
        else:
            # time-sliced logical clients: fold n_k * (theta_k - global) locally, then upload the mean
            # (DP: s_k * (theta_k - global) for every hosted client, even a single one, and the mean over clients;
            # robust: every hosted client uploads its own segment -- a median of per-rank sums is not a median of
            # clients)
            self.sync()
            fold = self.robust is None and (len(mine) > 1 or (self.dp is not None and mine))
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
                if self.personal is not None:
                    self.personal.swap_in(cid)
                ld = self._train_client(cid, X, y, n_epoch, first=(j == 0))
                if self.personal is not None:   # before the fold: it resets the replica, local range included
                    self.personal.swap_out(cid)
                nk = X.shape[0]
                losses_dev = ld * nk if losses_dev is None else losses_dev + ld * nk
                total_n += nk
                more = j + 1 < len(mine)               # the next co-resident client starts from the global model
                if self.robust is not None:
                    self.session.pack_client(j, reset=more)
                elif self.dp is not None:
                    self._dp_fold(j, more=more)
                elif self.topk is not None:
                    # top-k: one hosted client uploads its own list; several fold n_k * topk(u_k), then upload the
                    # folded mean's non-zero entries
                    if len(mine) == 1:
                        self.session.pack_topk(self._residual(cid))
                    else:
                        self.session.fold_topk(self._acc, self._residual(cid), nk, first=(j == 0), reset=more)
                elif len(mine) > 1:
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
                if self.topk is not None:
                    self.session.pack_nonzero()
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

    def _residual(self, cid: int) -> Optional[torch.Tensor]:
        return self.topk_state.residual(cid) if self.topk_state is not None else None

    def topk_residuals(self) -> Dict[int, torch.Tensor]:
        """``{client_id: e}``: the error-feedback residuals of the clients this rank hosts that have taken part so far
        (fp32 over the arena, on the engine's device; live, not copies).  Empty without error feedback."""
        if self.topk is None:
            raise RuntimeError("top-k uploads are off (compress=None)")
        self.sync()
        return dict(self.topk_state.e) if self.topk_state is not None else {}

    def last_upload_bytes(self) -> int:
        """Bytes this rank uploaded in the last round (a host read): the sparse list with ``compress='topk'`` (0 when it
        hosted no participant), else the dense wire."""
        self.sync()
        return self.session.last_upload_bytes() if self.topk is not None else self.session.wire_bytes()

    def last_krum(self) -> Dict[int, Tuple[float, bool]]:
        """``{client_id: (score, kept)}`` of the last Krum round's participants (a host read).  The session reports in
        segment order -- live ranks in order, then each rank's hosted participants in draw order -- and every rank
        knows the draw and who hosts whom, so every rank returns the same mapping."""
        if self.robust is None or self.robust.kind != "krum":
            raise RuntimeError("last_krum needs aggregator='krum'")
        if self._last_participants is None:
            raise RuntimeError("no round has run yet")
        _, scores, kept = self.session.last_krum()
        order = [c for r in range(self.world) for c in self._last_participants if c % self.world == r]
        if len(order) != len(scores):
            raise RuntimeError("the session reports {} clients, the round had {}".format(len(scores), len(order)))
        return {c: (float(scores[i]), bool(kept[i])) for i, c in enumerate(order)}

    def last_secagg_saturation(self) -> int:
        """Elements of this rank's upload that the last secure round clamped to ``[-secagg_range, secagg_range]`` or
        found non-finite (a device read, made only when asked)."""
        if self.secagg is None:
            raise RuntimeError("secure aggregation is off (secure_agg=False)")
        self.sync()
        return self.session.last_secagg_saturation()

    def server_state(self):
        """``(m, v)``: the server optimizer's state over the parameters (live fp32 tensors on the engine's device, equal
        on every rank; ``v`` is None for FedAvgM)."""
        self.sync()
        return self.session.server_state()

    def _train_client(self, cid: int, X, y, n_epoch: int, first: bool):
        """Local training of client ``cid`` on the replica; with SCAFFOLD, its correction before and its control-variate
        update after (before any fold resets the replica).  With augmentation, mixing or dropout, the client's stream of
        this round."""
        hp = self.hp
        if self.aug_hp is not None:
            hp = dict(hp, augment_stream=(self.n_rounds << 32) | int(cid), **self.aug_hp)
        if self.scaf is None:
            ld = self.trainer.run(X, y, n_epoch=n_epoch, return_device=True, **hp)
        else:
            self.scaf.begin_client(cid)
            ld = self.trainer.run(X, y, n_epoch=n_epoch, return_device=True, corr=self.scaf.corr, **hp)
            self.scaf.end_client(cid, self.arena, n_epoch * self.trainer.last_steps, self.hp["lr"], first=first)
        if self.trainer.grad_norms is not None:
            self._grad_norms[int(cid)] = self.trainer.grad_norms      # a fresh buffer per run: no copy
        return ld

    def last_grad_norms(self) -> Dict[int, List[List[float]]]:
        """``{client_id: [[norm per step] per epoch]}``: the pre-clip gradient norms of the clients this rank trained
        in the last round, logical clients included (a host read; empty when ``max_grad_norm`` is 0)."""
        return {c: t.tolist() for c, t in self._grad_norms.items()}

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
        """The round's one ``aggregate``: the loss, upload and stream arguments every kind of round takes, then the
        kind's own."""
        s = self.session
        kw = {}
        plain = self.robust is None and self.scaf is None and self.dp is None
        # a plain round of a rank that hosts no client (no loss) runs on the compute stream, with the kernel's own pack
        if isinstance(s, FedAvgSession) and not (plain and loss_dev is None):
            kw["on_side_stream"] = bool(self.overlap_collective)
            kw["prepacked"] = bool(self.prepack and getattr(self.trainer, "emitted_wire", False) and my_n > 0
                                   and not getattr(self.trainer, "last_had_tail_step", False))
        if loss_dev is not None and hasattr(s, "loss_local"):
            k = min(loss_dev.numel(), s.loss_local.numel())
            s.loss_local.zero_()
            s.loss_local[:k].copy_(loss_dev[:k])
        elif loss_dev is not None:
            kw["loss_history"] = loss_dev.tolist()
        if self.robust is not None:    # n_clients: segments packed by pack_client (logical clients), else seg 0 as usual
            if n_clients is not None:
                kw["n_clients"] = n_clients
        elif self.scaf is not None:    # SCAFFOLD: c += (sum of the ranks' dc) / N in the same collective
            kw["control"] = (self.scaf.c, self.scaf.up, self.logical_clients or self.world)
        elif self.dp is not None:
            kw["clipped"] = clipped
        s.aggregate(my_n=my_n, **kw)

    def global_loss(self, n_epoch: int) -> List[float]:
        return self.session.reduced_loss(n_epoch)

    # ------------------------------------------------------------------ evaluation
    def evaluate(self, shards, batch_size: Optional[int] = None) -> EvalResult:
        """Loss and accuracy of the global model on held-out data.  ``shards`` takes the forms of :meth:`run_round`:
        an ``(X, y)`` pair for this rank, a callable ``rank -> (X, y)``, or with logical clients a callable
        ``client_id -> (X, y)`` (every client this rank hosts is evaluated and the results are summed); ``None`` or
        an empty shard contributes nothing.  Host shards are staged into their own buffers, never the training ones.
        Nothing of the model, the arena or the training state changes.  Every rank must call it: the global numbers
        come from one all-reduce of ``[loss sum, #correct, n]`` over the session's process group.

        With ``local_keys``, each hosted client's shard is scored by that client's personalized model
        (:meth:`client_state_dict`; initial local values for a client that has not trained yet)."""
        self.sync()          # the round-end collective may still be writing the arena on its side stream
        batch = int(batch_size or self.hp["batch_size"])
        if self.logical_clients:
            ids = [c for c in range(self.logical_clients) if self.hosted(c)]
        else:
            ids = [self.rank]
        if shards is None:
            pairs = []
        elif self.logical_clients:
            pairs = [shards(c) for c in ids]
        else:
            pairs = [shards(self.rank) if callable(shards) else shards]
        saved = self._swap_for_eval() if self.personal is not None else None
        loss = correct = n = 0.0
        try:
            for cid, pair in zip(ids, pairs):
                if pair is None or pair[0].shape[0] == 0:
                    continue
                X, y = pair
                if self.device.type == "cuda" and not X.is_cuda:
                    # one staging buffer per shape: a pass ends with a host read, so the next shard may overwrite it
                    X, y = self._copy_in(self._eval_stage, X, y, 0)
                if saved is not None:
                    self._load_local(self.personal.values(cid))
                ls, c, k = self.trainer.evaluate(X, y, batch_size=batch)
                loss, correct, n = loss + ls, correct + c, n + k
        finally:
            if saved is not None:
                a, (lo, hi) = self.arena, self.arena.local_range
                a.theta[lo:hi].copy_(saved[0])
                if saved[1] is not None:
                    a.theta_bf16[lo:hi].copy_(saved[1])
        tot = [loss, correct, n]
        group = getattr(self.session, "group", None)
        if self.world > 1 and torch.distributed.is_available() and torch.distributed.is_initialized():
            t = torch.tensor(tot, dtype=torch.float64, device=self.device)
            torch.distributed.all_reduce(t, group=group)
            tot = t.tolist()
        return EvalResult(loss=_mean(tot[0], tot[2]), accuracy=_mean(tot[1], tot[2]), n_samples=int(tot[2]),
                          local_loss=_mean(loss, n), local_accuracy=_mean(correct, n), local_n_samples=int(n))

    def _swap_for_eval(self):
        a, (lo, hi) = self.arena, self.arena.local_range
        return a.theta[lo:hi].clone(), a.theta_bf16[lo:hi].clone() if a.theta_bf16 is not None else None

    @torch.no_grad()
    def _load_local(self, v: torch.Tensor) -> None:
        """Put one client's local entries into the replica's theta and bf16 shadow (evaluation only)."""
        a, (lo, hi) = self.arena, self.arena.local_range
        a.theta[lo:hi].copy_(v)
        if a.theta_bf16 is not None:
            a.theta_bf16[lo:hi].copy_(v)

    def _check_hosted(self, cid: int) -> None:
        if self.personal is None:
            raise RuntimeError("client-local entries are off (local_keys=None)")
        if not (0 <= int(cid) < (self.logical_clients or self.world)) or not self.hosted(int(cid)):
            raise RuntimeError("client {} is not hosted by rank {}".format(cid, self.rank))

    def local_entries(self, cid: int) -> Dict[str, torch.Tensor]:
        """``{key: tensor}`` copies of hosted client ``cid``'s local entries (the initial values until it has trained)."""
        self._check_hosted(cid)
        self.sync()
        return self.personal.entries(cid)

    def client_state_dict(self, cid: int):
        """The personalized model of hosted client ``cid`` (copies): the shared entries of the current global model and
        the client's local entries."""
        self._check_hosted(cid)
        self.sync()
        sd = self.model.state_dict()
        mine = self.personal.entries(cid)
        return type(sd)((k, mine[k] if k in mine else v.clone()) for k, v in sd.items())

    def state_dict(self):
        """The global model (live views of the arena).  With ``local_keys`` its local entries are copies of their
        initial values: what a client that has not trained yet starts from."""
        self.sync()
        sd = self.model.state_dict()
        if self.personal is None:
            return sd
        init = self.personal.initial_entries()
        return type(sd)((k, init[k] if k in init else v) for k, v in sd.items())
