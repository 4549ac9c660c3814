"""The fused NVLink FedAvg data plane (host side).

``FedAvgSession`` owns the symmetric wire buffer of one rank and launches the
single-kernel round-end collective (``csrc/fedavg.cu``): pack/cast -> weighted
reduce over peer memory -> broadcast -> running-mean apply into the fp32 master,
the bf16 shadow and (optionally) per-tile arrival flags that gate the first GEMM
of the next forward (``bcast_gemm``).

It replaces, for GPU-seated clients, the reference's upload (worker.py:108-118),
the manager's CPU reduce (manager.py:119-126), the broadcast (manager.py:77-86)
and ``load_state_dict`` (worker.py:98).  ``NcclSession`` implements the same
interface with ``torch.distributed`` collectives: it is the BASELINE the fused
kernel is measured against and the oracle the tests compare with -- not the
product path.

Both take ``dp=DPConfig(...)`` (``parallel/dp.py``): DP-FedAvg, the clipped uniform mean of the participants' updates
plus Gaussian noise on the sum.  The fused session clips with one deterministic norm kernel per round on the
collective's stream, publishes the factor in a small per-rank CLIP PAGE of the symmetric buffer, and the collective
applies it on the reader side and adds the noise in the tile owner's fp32 accumulator; DP rounds always run on peer
loads (the switch of NVLS adds raw wire values, before the factors are known).

Both take ``scaffold=True`` (SCAFFOLD, ``parallel/scaffold.py``): every round then also carries the control-variate
update, ``aggregate(control=(c, dc, N))`` -- ``c += (sum over ranks of dc) / N``.  The fused session lays out each
parity half of its wire as ``[segment 0 | pad | segment 1]`` (segment 1: ``dc`` over the parameters, in the session's
wire format) and the collective reduces both segments in one launch, on peer loads.

Both take ``robust=RobustConfig(...)`` (``parallel/robust.py``): the round's update is the coordinate-wise median or
trimmed mean of the participating CLIENTS' deltas instead of the weighted mean.  A median of per-rank sums is not a
median of clients, so every hosted client uploads its own segment: ``max_clients=S`` lays out each parity half of the
fused session's wire as ``[seg 0 | pad | seg 1 | ... | seg S-1]`` (``S = 1`` is the plain layout), ``pack_client(j)``
fills segment ``j`` and ``aggregate(..., n_clients=m)`` runs the robust kernel over the ``m`` segments of every rank
(their counts travel in a per-rank page), always on peer loads.

``robust=RobustConfig("krum", krum_f=f, krum_m=m)`` selects Multi-Krum: the fused session then also allocates a
per-rank DISTANCE PAGE (4 KB per round parity) through which the ranks exchange their partial pair distances inside the
collective, and :meth:`last_krum` returns the last round's distances, scores and kept clients in segment order.

Both take ``topk=TopKConfig(ratio, error_feedback)`` (``parallel/compress.py``): every participating client uploads only
its ``k`` largest-magnitude update entries (the rest carried in its residual).  Each parity half of the fused session's
wire is then ``[seg 0: the dense result | pad | sparse segment]``, the sparse segment being ``uint32 rowptr[n / 1024 +
1] | pad | uint16 off[cap] | pad | values[cap]`` in the wire dtype (fp32 or bf16).  :meth:`pack_topk` selects and
compacts one client into it, :meth:`fold_topk` folds a co-resident logical client's selection into an accumulator and
:meth:`pack_nonzero` compacts the folded mean; the collective's owners add the lists into a shared-memory tile on peer
loads (the switch cannot add sparse lists).  ``cap = k``, or ``min(n, max_clients * k)`` for ``max_clients`` folded
clients.  The optimizer-emitted upload is off: the selection needs all of ``u``.

Both take ``server_opt=ServerOptConfig(...)`` (``parallel/server_opt.py``): FedAvgM, FedAdagrad, FedYogi or FedAdam
applied to the round's aggregate, whatever computed it (mean, DP, SCAFFOLD, median, trimmed mean, Krum).  The session
allocates the state ``arena.server_m`` / ``arena.server_v`` over the parameters, replicated on every rank; the fused
session runs the round's kernel on ``ServerOptArgs<...>`` of the round's arguments, whose apply phase takes the step, and
:class:`NcclSession` calls :func:`server_step_` where it would add the aggregate.  :meth:`server_state` reads the state.

Both take ``secagg=SecAggConfig(range)`` (``parallel/secagg.py``): secure aggregation over the fp32-sized wire in delta
mode.  The ranks agree on pairwise ChaCha20 keys with one X25519 exchange at construction; every round each participant
uploads its fixed-point update plus its pairwise masks, which cancel in the uint32 sum.  The fused session runs the
``Agg::secagg`` kernel (count barrier, masked pack, wrapping reduce, decode in the apply phase), always on peer loads and
never prepacked; :class:`NcclSession` encodes with the same kernel (the numpy reference on the CPU), all-reduces the
masked words as int64 and keeps the low 32 bits.  :meth:`last_secagg_saturation` reads this rank's clamped elements of
the last round.
"""
from __future__ import annotations

from typing import List, Optional, Sequence

import numpy as np
import torch

from .arena import ParamArena
from .compress import TopKConfig, n_float, sparse_upload_bytes, topk_ef_
from .dp import DPConfig, clip_factor, normals
from .features import check_features, peer_loads_only
from .robust import MAX_ROBUST_CLIENTS, RobustConfig, krum_select, robust_combine
from . import secagg as sa
from .secagg import SecAggConfig
from .server_opt import ServerOptConfig, apply_update_
from .symm import SymmetricBuffer

MAX_LOSS = 64       # per-epoch loss slots carried through the collective
MAX_CTAS = 296      # pad slots; the kernel runs one 512-thread CTA per SM (132 on H100 SXM), clamped by the launcher


def _align(x: int, a: int) -> int:
    return (x + a - 1) // a * a


def _session_rules(features: dict, dp: Optional[DPConfig], robust: Optional[RobustConfig]) -> None:
    """:func:`check_features` for a session's features with a round's ``dp`` / ``robust``, after ``TypeError`` for a
    ``robust``, ``topk`` or ``server_opt`` that is not its configuration class."""
    for x, cls, name in ((robust, RobustConfig, "robust"), (features["topk"], TopKConfig, "topk"),
                         (features["server_opt"], ServerOptConfig, "server_opt"), (features["secagg"], SecAggConfig,
                                                                                   "secagg")):
        if x is not None and not isinstance(x, cls):
            raise TypeError("{}= takes a {}".format(name, cls.__name__))
    f = dict(features)
    check_features(dp=dp, robust=robust, secure_agg=f.pop("secagg") is not None, **f)


def _init_session(arena: ParamArena, features: dict, dp: Optional[DPConfig], robust: Optional[RobustConfig],
                  max_clients: int) -> int:
    """Check a session's features (either kind of session), allocate the server optimizer's fresh state in the arena
    (``m = 0``, ``v = tau^2``) and return the client segments per rank."""
    _session_rules(features, dp, robust)
    if features["local"] != (arena.local_range is not None):
        raise ValueError("local=True needs an arena built with local entries, and such an arena needs local=True")
    if robust is not None:
        if not (1 <= int(max_clients) <= MAX_ROBUST_CLIENTS):
            raise ValueError("max_clients must be in 1..{}, got {!r}".format(MAX_ROBUST_CLIENTS, max_clients))
    elif features["topk"] is not None:      # the folded clients' union of supports sizes the sparse segment
        if int(max_clients) < 1:
            raise ValueError("max_clients must be >= 1, got {!r}".format(max_clients))
    elif int(max_clients) != 1:
        raise ValueError("max_clients > 1 needs a robust aggregator: plain rounds fold their clients into one upload")
    server_opt = features["server_opt"]
    if server_opt is not None:
        arena.server_m, arena.server_v = server_opt.init_state(arena.n_param, arena.device)
    return int(max_clients)


def _check_control(scaffold: bool, control) -> None:
    if scaffold and control is None:
        raise ValueError("a SCAFFOLD session needs control=(c, dc, n_clients) every round")
    if not scaffold and control is not None:
        raise ValueError("control= needs a session built with scaffold=True")


def _secagg_keys(secagg: Optional[SecAggConfig], group) -> dict:
    """``{peer rank: eight uint32 key words}`` of a secure session (one X25519 exchange over ``group``), else ``{}``."""
    if secagg is None:
        return {}
    return {j: sa.key_words(k) for j, k in sa.agree_keys(group).items()}


def _agree_seed(dp: Optional[DPConfig], group) -> Optional[DPConfig]:
    """Every rank must draw the same noise: take rank 0's Philox key (a DPConfig built with seed=None differs per
    process)."""
    import torch.distributed as dist
    if dp is None or not (dist.is_available() and dist.is_initialized()) or dist.get_world_size(group) == 1:
        return dp
    box = [dp.seed]
    src = dist.get_global_rank(group, 0) if group is not None else 0
    dist.broadcast_object_list(box, src=src, group=group)
    return DPConfig(dp.clip, dp.noise_multiplier, seed=int(box[0]))


class FedAvgSession:
    def __init__(self, arena: ParamArena, group=None, *, wire_dtype: str = "bf16", mode: str = "delta",
                 nvls: "bool | str" = "auto", n_ctas: Optional[int] = None, tile_elems: int = 0, timeout_log2: int = 24,
                 reset_momentum: bool = True, tile_flags: bool = False, dp: Optional[DPConfig] = None,
                 scaffold: bool = False, robust: Optional[RobustConfig] = None, max_clients: int = 1,
                 server_opt: Optional[ServerOptConfig] = None, topk: Optional[TopKConfig] = None,
                 local: bool = False, secagg: Optional[SecAggConfig] = None):
        from ..ops._ext import load
        self._C = load()
        assert wire_dtype in ("bf16", "fp32", "fp8") and mode in ("delta", "weights")
        self._features = dict(wire_dtype=wire_dtype, mode=mode, scaffold=scaffold, topk=topk, server_opt=server_opt,
                             tile_flags=tile_flags, local=bool(local), secagg=secagg,
                              frozen=arena.frozen_range is not None)
        self.max_clients = _init_session(arena, self._features, dp, robust, max_clients)
        self.local_range = arena.skip_range    # client-local or frozen: the range the round never touches
        self.n_wire = arena.n_shared           # elements on the wire: the arena minus that range
        self.topk, self.server_opt = topk, server_opt
        self._sopt_coef = list(server_opt.coefficients()) if server_opt is not None else []
        self.robust = robust
        self.krum = robust is not None and robust.kind == "krum"
        self.scaffold = bool(scaffold)
        self.arena = arena
        self.device = arena.device
        self.group = group
        self.wire_dtype = wire_dtype
        self.wire_bf16 = wire_dtype == "bf16"
        self.wire_kind = {"fp32": 0, "bf16": 1, "fp8": 2}[wire_dtype]
        self.delta = mode == "delta"
        if n_ctas is None:   # one CTA per SM: the cooperative launch clamps the grid to what is co-resident
            dev = torch.device(self.device)
            n_ctas = torch.cuda.get_device_properties(dev).multi_processor_count if dev.type == "cuda" else 1
        self.n_ctas = max(1, min(int(n_ctas), MAX_CTAS))
        self.tile_elems = int(tile_elems)
        # every cross-GPU spin is BOUNDED by default (2^24 polls, several seconds): a seat that dies between the
        # manager's plan and its launch turns into an error status on the survivors (check()), not into eight GPUs
        # spinning forever -- the NCCL failure mode this data plane exists to avoid.  0 = spin without limit.
        self.timeout_log2 = int(timeout_log2)
        self.reset_momentum = reset_momentum
        # wire / int / loss pages exist TWICE (round parity): the kernel has no closing barrier, a rank that races ahead
        # packs the next round into the other half while a slow peer still applies this one (csrc/fedavg.cu)
        # SCAFFOLD: segment 1 (dc over the parameters) starts at seg1_off of each half
        self.seg1_off = _align(self._seg_bytes(arena.n), 256) if self.scaffold else 0
        # robust: S client segments per half, seg_stride bytes apart (2 * S * seg_stride bytes of symmetric memory)
        self.seg_stride = _align(self._seg_bytes(arena.n), 256)
        half = self.max_clients * self.seg_stride if robust is not None else self.wire_bytes()
        if self.topk is not None:
            if arena.n % self.FLAG_GRANULE:
                raise ValueError("top-k uploads need an arena of whole 1024-element granules")
            self.topk_k = self.topk.k(n_float(arena))
            self.topk_cap = min(arena.n, self.max_clients * self.topk_k)
            self.topk_rowptr_off = _align(self._seg_bytes(arena.n), 256)
            self.topk_off_off = self.topk_rowptr_off + _align(4 * (arena.n // self.FLAG_GRANULE + 1), 256)
            self.topk_val_off = self.topk_off_off + _align(2 * self.topk_cap, 256)
            half = self.topk_val_off + self.topk_cap * (4 if wire_dtype == "fp32" else 2)
        self.half_wire = _align(half, 2 << 20)                        # multicast-friendly granularity
        self.half_int = _align(max(arena.n_int, 1) * 8, 256)
        self.half_loss = _align(MAX_LOSS * 4, 256)
        self.half_clip = 256                                          # DP: this rank's clip factor s_r; robust: m_r
        # Krum: this rank's fp64 pair distances of the round (496 at P = 32); only Krum sessions have the page
        self.half_dist = _align(self._C.KRUM_PAIRS * 8, 4096) if self.krum else 0
        self.off_wire = 0
        self.off_int = 2 * self.half_wire
        self.off_loss = self.off_int + 2 * self.half_int
        self.off_clip = self.off_loss + 2 * self.half_loss
        self.off_dist = self.off_clip + 2 * self.half_clip
        self.off_pads = _align(self.off_dist + 2 * self.half_dist, 256)
        total = _align(self.off_pads + (MAX_CTAS + 8) * self._C.MAX_RANKS * 8, 2 << 20)
        self.symm = SymmetricBuffer(total, self.device, group)
        self.rank, self.world = self.symm.rank, self.symm.world
        assert self.world <= self._C.MAX_RANKS
        # nvls: True, False or "auto" (on where the box has multicast; autotuned below)
        self.use_nvls = bool(nvls and self.symm.has_multicast
                             and not peer_loads_only(wire_dtype=wire_dtype, dp=dp, scaffold=scaffold, robust=robust,
                                                     topk=topk, secure_agg=secagg is not None))
        self.dp = _agree_seed(dp, group)
        # secure aggregation: the pair keys (host memory and this rank's kernel arguments only) and the saturation count
        self.secagg = secagg
        if secagg is not None:
            if arena.n >= sa.MAX_ARENA:
                raise ValueError("secure aggregation needs an arena of fewer than 2^36 elements")
            keys = _secagg_keys(secagg, group)
            self._secagg_words = [w for r in range(self.world) for w in keys.get(r, [0] * 8)]
            self.secagg_sat = torch.zeros(1, dtype=torch.int64, device=self.device)
        self._topk_work = None          # top-k: the selection's scratch, the residual-less u, the last upload's row end
        self._topk_u = None
        self._topk_end = None
        self._topk_sent = None
        self._packed_epoch = None   # robust: barrier epoch whose wire half pack_client filled
        if self.krum:   # the rank step's per-CTA partials and counters, and the host report (csrc/launch.h)
            self.krum_work = torch.zeros(self._C.KRUM_MAX_CTAS * self._C.KRUM_PAIRS, dtype=torch.float64,
                                         device=self.device)
            self.krum_sync = torch.zeros(2, dtype=torch.int32, device=self.device)
            self.krum_report = torch.zeros(self._C.KRUM_REPORT, dtype=torch.float64, device=self.device)
        # DP bookkeeping: norm-kernel partials, the last clip factor / norm of this rank, non-finite updates so far
        self.dp_work = torch.zeros(self._C.DP_WORK_WORDS, dtype=torch.int64, device=self.device)
        self.dp_s = torch.ones(1, dtype=torch.float32, device=self.device)
        self.dp_norm = torch.zeros(1, dtype=torch.float32, device=self.device)
        self.dp_nonfinite = torch.zeros(1, dtype=torch.int32, device=self.device)
        self.epoch = 0
        self.rounds = 0
        self.stale = False          # True after a round this seat sat out: its weights are no longer the global model
        self.status = torch.zeros(1, dtype=torch.int32, device=self.device)
        self.loss_local = torch.zeros(MAX_LOSS, dtype=torch.float32, device=self.device)
        self.loss_out = torch.zeros(MAX_LOSS, dtype=torch.float32, device=self.device)
        # tile_elems == 0: sized per launch so that every CTA of every live rank owns ~one tile
        self.min_tile = 1024
        n_tiles = (arena.n + self.min_tile - 1) // self.min_tile
        self.tile_flags = torch.zeros(n_tiles, dtype=torch.int32, device=self.device) if tile_flags else None
        # flag value consumers must wait for (= rounds launched so far): device-resident so captured graphs follow
        self.epoch_word = torch.zeros(1, dtype=torch.int32, device=self.device)
        self.last_tile_elems = self.tile_elems or self.min_tile
        # a high-priority stream lets the collective's CTAs become resident ahead of a flag-gated
        # GEMM that is launched right behind it on the compute stream
        self.stream = torch.cuda.Stream(device=self.device, priority=-1) if self.device.type == "cuda" else None
        self.symm.barrier()
        # K4: the last SGD step of an epoch may write this rank's wire copy itself (ops.fused_sgd(pack=...)); the wire
        # address of the upcoming round (parity half) and the pack scale live in device words so a captured graph follows
        self.wire_slot = torch.zeros(1, dtype=torch.int64, device=self.device)
        self.pack_scale = torch.ones(1, dtype=torch.float32, device=self.device)
        self._armed_for = None     # (epoch, scale) the wire words were armed for
        self.phase_ns = None       # enable_phase_timing(): int64[16] of %globaltimer stamps written by the kernel
        self.nvls_choice = "forced" if nvls != "auto" else "default"
        if nvls == "auto" and self.use_nvls and self.delta and self.world > 1 and arena.global_w is not None:
            self.autotune_nvls()
        # barrier epoch at the end of construction (the autotune above already ran collectives): identical on every rank,
        # and the origin of the manager-dictated round index (aggregate(round_index=...))
        self.base_epoch = self.epoch

    FLAG_GRANULE = 1024        # elements per arrival flag (csrc/fedavg.cu)

    PHASES = ("pack", "barrier1", "reduce_bcast", "barrier2", "apply", "exit")

    def enable_phase_timing(self) -> None:
        """Ask the kernel to record %globaltimer at its phase boundaries (first and last CTA) -- the way to
        see where a multi-GPU round goes, since kernels with cross-GPU spin barriers cannot run under ncu.
        Needs an extension built with ``BATON_BUILD_PHASE_TIMING=1 python -m baton_b200.build_ext`` (the default
        build compiles the stamps out, so all durations read 0)."""
        self.phase_ns = torch.zeros(16, dtype=torch.int64, device=self.device)

    def phase_breakdown_us(self) -> dict:
        """Phase durations of the LAST launch in microseconds: ``{"first_cta": {...}, "last_cta": {...}}``."""
        if self.phase_ns is None:
            return {}
        t = self.phase_ns.tolist()
        out = {}
        for name, base in (("first_cta", 0), ("last_cta", 8)):
            out[name] = {p: (t[base + i + 1] - t[base + i]) / 1e3 for i, p in enumerate(self.PHASES)}
        return out

    def autotune_nvls(self, iters: int = 3) -> None:
        """Measure, don't guess: time the collective both ways (peer loads/stores vs in-switch
        ``multimem`` reduce + multicast store) on THIS box and world size and keep the faster one.  Runs on
        zero deltas (``theta == global`` right after the arena is built), so it leaves the model untouched;
        every rank takes the max over ranks, so all ranks agree."""
        import torch.distributed as dist
        if not torch.equal(self.arena.theta[: self.arena.n_param], self.arena.global_w[: self.arena.n_param]):
            return                                   # replicas already drifted: keep the default
        best = {}
        sopt, self.server_opt = self.server_opt, None    # zero deltas must not step the server optimizer's state
        try:
            best = self._time_nvls_modes(iters)
        finally:
            self.server_opt = sopt
        t = torch.tensor([best[False], best[True]], device=self.device, dtype=torch.float64)
        dist.all_reduce(t, op=dist.ReduceOp.MAX, group=self.group)
        self.use_nvls = bool(t[1] < t[0])
        self.nvls_choice = "autotuned p2p {:.0f} us vs nvls {:.0f} us".format(float(t[0]) * 1e3, float(t[1]) * 1e3)
        self.check()
        self.symm.barrier()

    def _time_nvls_modes(self, iters: int) -> dict:
        best = {}
        for mode in (False, True):
            self.use_nvls = mode
            ts = []
            for it in range(iters + 1):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                self.aggregate(my_n=1.0)
                e1.record()
                torch.cuda.synchronize(self.device)
                if it:
                    ts.append(e0.elapsed_time(e1))
            best[mode] = min(ts)
        return best

    # ------------------------------------------------------------------ K4: upload copy emitted by the optimizer
    def pack_spec(self) -> Optional[dict]:
        """Arguments for ``ops.fused_sgd(pack=...)`` (stable device tensors: safe to capture), or None when the wire
        format needs the in-kernel pack (block-scaled fp8)."""
        if (self.wire_kind == 2 or self.device.type != "cuda" or self.topk is not None or self.local_range is not None
                or self.secagg is not None):
            return None
        a = self.arena
        return {"wire_slot": self.wire_slot, "global_w": a.global_w if self.delta else None, "scale": self.pack_scale,
                "n_pack": a.n, "wire_fp32": self.wire_kind == 0}

    def arm_prepack(self, my_n: float) -> None:
        """Point the device words at the wire half of the UPCOMING round and set the pack scale (n_k under NVLS, where
        the switch can only add; 1 for peer loads, which weight on the reader side).  Call before the local epoch(s)."""
        par = (self.epoch // 3) & 1
        addr = self.symm.peer_ptrs(self.off_wire + par * self.half_wire)[self.rank]
        scale = float(my_n) if (self.use_nvls and self.world > 1) else 1.0
        key = (self.epoch, scale)
        if self._armed_for != key:
            self.wire_slot.fill_(int(addr))
            self.pack_scale.fill_(scale)
            self._armed_for = key

    # ------------------------------------------------------------------ robust rounds: one segment per client
    def segment_ptr(self, j: int) -> int:
        """Device address of client segment ``j`` of this rank's wire half for the upcoming round."""
        par = (self.epoch // 3) & 1
        return self.symm.peer_ptrs(self.off_wire + par * self.half_wire)[self.rank] + int(j) * self.seg_stride

    def pack_client(self, j: int, reset: bool = False) -> None:
        """Upload the replica's client into segment ``j`` of the upcoming round: ``seg_j = cast(theta - global)`` in
        the wire format (the collective's own pack, fp8 block scales included).  ``reset``: also return the replica
        to the global model (theta, bf16 shadow, momentum) for the next hosted client.  Runs on the current stream."""
        if self.robust is None:
            raise RuntimeError("pack_client needs a session built with robust=")
        if not (0 <= int(j) < self.max_clients):
            raise ValueError("segment {} out of range (max_clients={})".format(j, self.max_clients))
        a = self.arena
        self._C.pack_client(self.segment_ptr(j), a.theta, a.global_w, a.theta_bf16,
                            a.momentum if reset else None, self.wire_kind, bool(reset))
        self._packed_epoch = self.epoch

    # ------------------------------------------------------------------ top-k rounds: sparse uploads
    def _topk_lists(self):
        if self.topk is None:
            raise RuntimeError("top-k uploads need a session built with topk=")
        if self._topk_work is None:
            from ..ops import functional as F
            self._topk_work = F.topk_work(self.arena.n, self.device)
        base = self.segment_ptr(0)
        par = (self.epoch // 3) & 1
        self._topk_end = (self.epoch, self.off_wire + par * self.half_wire + self.topk_rowptr_off
                          + 4 * (self.arena.n // self.FLAG_GRANULE))
        return base + self.topk_rowptr_off, base + self.topk_off_off, base + self.topk_val_off

    def _topk_residual(self, e: Optional[torch.Tensor]) -> torch.Tensor:
        if self.topk.error_feedback:
            if e is None or e.dtype != torch.float32 or e.numel() != self.arena.n:
                raise ValueError("error feedback needs the client's fp32 residual over the arena")
            return e
        if self._topk_u is None:
            self._topk_u = torch.empty_like(self.arena.theta)
        return self._topk_u

    def pack_topk(self, e: Optional[torch.Tensor] = None) -> None:
        """Upload the replica's client as its top-k list for the upcoming round: ``u = (theta - global) + e``, the ``k``
        largest ``|u|`` into the sparse segment, ``e`` = the rest (``e``: the client's residual, required with error
        feedback and ignored without).  Runs on the current stream."""
        from ..ops import functional as F
        a = self.arena
        u = self._topk_residual(e)
        rowptr, off, val = self._topk_lists()
        F.topk_pack(a.theta, a.global_w, u, self.topk_k, self._topk_work, rowptr, off, val,
                    ef=self.topk.error_feedback, wire_fp32=self.wire_kind == 0, cap=self.topk_cap)
        self._packed_epoch = self.epoch

    def fold_topk(self, acc: torch.Tensor, e: Optional[torch.Tensor], nk: float, first: bool, reset: bool) -> None:
        """A co-resident logical client: ``acc (+)= nk * topk(u)`` (``first``: from 0), its residual updated, and
        (``reset``) the replica returned to the global model for the next one.  :meth:`pack_nonzero` uploads the fold."""
        from ..ops import functional as F
        a = self.arena
        u = self._topk_residual(e)
        if self._topk_work is None:
            self._topk_work = F.topk_work(a.n, self.device)
        F.topk_fold(a.theta, a.global_w, u, self.topk_k, self._topk_work, acc, nk, ef=self.topk.error_feedback,
                    first=first, reset=reset, w_bf16=a.theta_bf16, momentum=a.momentum)

    def pack_nonzero(self) -> None:
        """Upload ``theta - global`` where it is non-zero (the folded mean of the hosted clients: at most ``cap``
        entries, the union of their supports)."""
        from ..ops import functional as F
        a = self.arena
        rowptr, off, val = self._topk_lists()
        F.nonzero_pack(a.theta, a.global_w, self._topk_work, rowptr, off, val, wire_fp32=self.wire_kind == 0,
                       cap=self.topk_cap)
        self._packed_epoch = self.epoch

    def last_upload_entries(self) -> int:
        """Entries of this rank's upload in the last top-k round (a host read; 0 when it sent none)."""
        if self.topk is None:
            raise RuntimeError("last_upload_entries needs a session built with topk=")
        if self._topk_sent is None:
            return 0
        self.join()
        return int(self.symm.view(self._topk_sent, 1, torch.int32).item())

    def last_upload_bytes(self) -> int:
        """Bytes of this rank's upload in the last round: the sparse list of a top-k round, else :meth:`wire_bytes`."""
        if self.topk is None:
            return self.wire_bytes()
        if self._topk_sent is None:
            return 0
        return sparse_upload_bytes(self.arena.n, self.last_upload_entries(), self.wire_dtype)

    # ------------------------------------------------------------------ the collective
    def aggregate(self, n_samples_by_rank: Optional[Sequence[float]] = None,
                  alive_ranks: Optional[Sequence[int]] = None, my_n: Optional[float] = None,
                  loss_history: Optional[Sequence[float]] = None, on_side_stream: bool = False,
                  round_index: Optional[int] = None, prepacked: bool = False, dp: Optional[DPConfig] = None,
                  clipped: bool = False, control=None, n_clients: Optional[int] = None,
                  robust: Optional[RobustConfig] = None) -> None:
        """Launch the fused reduce+broadcast+apply.  Either the full per-rank sample
        counts are given (manager-driven rounds: the plan comes over HTTP) or only this
        rank's own count ``my_n`` (SPMD engine: peers' counts ride on the barrier flags).

        ``round_index``: number of aggregations the MANAGER has dispatched before this one.  The manager is the single
        authority for it: the barrier epoch becomes ``base_epoch + 3 * round_index`` on every seat, so a seat that sat
        out rounds (evicted, re-registered) re-enters in step with its peers instead of racing them with a lagging
        counter (epochs must never run backwards: the pads keep the highest epoch ever seen).

        ``dp`` (default: the session's): a DP-FedAvg round.  The counts must then be CLIENTS per rank (1 for a plain
        seat), not samples, and every rank must pass the same ``dp`` (the manager's plan carries it; a session built
        with ``dp=`` agreed on rank 0's key at construction).  ``clipped=True``: this rank's upload is already a sum of clipped updates divided by its
        count (logical clients folded with :func:`ops.functional.fold_client_scaled`), so its clip factor is 1.

        ``control = (c, dc, n_clients)`` (every round of a ``scaffold=True`` session, and only there): SCAFFOLD's
        server control-variate update in the same launch -- ``c += (sum over participating ranks of dc) / n_clients``
        on every live rank.  ``c`` and ``dc`` are fp32 over the arena's parameters; ``dc`` is this rank's summed client
        updates (read only when this rank participates).  The optimizer-emitted upload (``prepacked``) covers the
        model segment only.

        ``n_clients`` (sessions built with ``robust=``): the number of client segments this rank contributes, filled by
        :meth:`pack_client` for this round (default: 1 when this rank's count is non-zero, packed by the kernel or by
        the optimizer).  The robust kernel then combines the segments of every live rank.  ``robust`` (default: the
        session's): a robust round on any delta-mode session without arrival flags, one segment per rank (the seated
        planes' plan carries it)."""
        world = self.world
        dp = dp if dp is not None else self.dp
        robust = robust if robust is not None else self.robust
        if dp is not self.dp or robust is not self.robust:     # the session's own features were checked when built
            _session_rules(self._features, dp, robust)
        _check_control(self.scaffold, control)
        if robust is None and n_clients is not None:
            raise ValueError("n_clients= needs a robust session or robust=")
        if robust is not None and robust.kind == "krum" and not self.krum:
            raise ValueError("a Krum round needs a session built with robust=RobustConfig('krum', ...): the ranks "
                             "exchange their distances through a page only Krum sessions allocate")
        if round_index is not None:
            self.epoch = (self.base_epoch + 3 * int(round_index)) & 0xFFFFFFFF
        if n_samples_by_rank is not None:
            counts = [float(x) for x in n_samples_by_rank] + [0.0] * (world - len(n_samples_by_rank))
            counts = counts[:world]
            from_flags = False
        else:
            assert my_n is not None
            counts = [0.0] * world
            counts[self.rank] = float(my_n)
            from_flags = True
        alive = list(range(world)) if alive_ranks is None else [int(r) for r in alive_ranks if 0 <= int(r) < world]
        if self.rank not in alive:
            # not part of this round: the replica goes stale (``stale`` tells the worker to pull the global model
            # before it takes part again) but the barrier epoch and the round counter keep pace with the peers
            self.epoch = (self.epoch + 3) & 0xFFFFFFFF
            self.rounds += 1
            self.stale = True
            return
        mask = 0
        for r in alive:
            mask |= 1 << r
        if loss_history is not None:
            k = min(len(loss_history), MAX_LOSS)
            self.loss_local.zero_()
            self.loss_local[:k].copy_(torch.tensor([float(x) for x in loss_history[:k]]), non_blocking=True)
        a = self.arena
        # the optimizer's wire copy is only valid for the round / scale it was armed for and when the collective runs
        # the way arm_prepack assumed (NVLS needs every rank alive); otherwise the kernel packs itself (always correct)
        nvls_now = bool(self.use_nvls and len(alive) == world
                        and not peer_loads_only(wire_dtype=self.wire_dtype, dp=dp, scaffold=self.scaffold,
                                                robust=robust, topk=self.topk))
        want_scale = (counts[self.rank] if not from_flags else float(my_n)) if (self.use_nvls and world > 1) else 1.0
        prepacked = bool(prepacked and self.wire_kind != 2 and self._armed_for == (self.epoch, float(want_scale))
                         and (nvls_now == bool(self.use_nvls and world > 1)) and self.secagg is None)
        if robust is not None:
            m = (1 if counts[self.rank] != 0.0 else 0) if n_clients is None else int(n_clients)
            if not (0 <= m <= self.max_clients):
                raise ValueError("n_clients={} outside 0..max_clients={}".format(m, self.max_clients))
            if n_clients is not None and m > 0:
                if self._packed_epoch != self.epoch:
                    raise RuntimeError("the client segments were not packed for this round (pack_client before "
                                       "aggregate, with the same round index)")
                prepacked = True
            self._packed_epoch = None
        self.last_prepacked = prepacked
        if self.tile_elems:
            tile = self.tile_elems
        else:   # one tile per (live rank, CTA): n / (A * G), rounded up to a multiple of 8 elements
            per = -(-self.n_wire // (len(alive) * self.n_ctas))
            tile = max(self.min_tile, (per + 31) // 32 * 32)
        if self.tile_flags is not None or self.topk is not None:
            # arrival flags and sparse rows cover fixed 1024-element granules: tiles must not split one
            tile = (tile + self.FLAG_GRANULE - 1) // self.FLAG_GRANULE * self.FLAG_GRANULE
        self.last_tile_elems = tile
        flag_value = self.rounds + 1
        par = (self.epoch // 3) & 1            # round parity: which half of the wire / int / loss / clip pages this round uses
        o_wire, o_int, o_loss = (self.off_wire + par * self.half_wire, self.off_int + par * self.half_int,
                                 self.off_loss + par * self.half_loss)
        o_clip = self.off_clip + par * self.half_clip
        cur = torch.cuda.current_stream(self.device)
        stream = self.stream if on_side_stream else cur
        if self.tile_flags is not None:
            self.epoch_word.fill_(flag_value)       # compute stream: whatever is enqueued after this call waits for THIS round
        if on_side_stream:
            stream.wait_stream(cur)
        if self.topk is not None:
            if counts[self.rank] != 0.0 and self._packed_epoch != self.epoch:
                raise RuntimeError("a top-k round needs this rank's upload packed for it (pack_topk or pack_nonzero "
                                   "before aggregate, with the same round index)")
            self._topk_sent = self._topk_end[1] if counts[self.rank] != 0.0 else None
            self._packed_epoch = None
            prepacked = True        # the sparse lists are written before the launch: a top-k round has no pack phase
        # the arguments every kind of round takes (csrc/bindings.cpp), then the kind's own
        common = (self.symm.peer_ptrs(o_wire), self.symm.peer_ptrs(self.off_pads),
                  self.symm.mc(o_wire) if nvls_now else 0,
                  a.theta, a.global_w, a.theta_bf16, a.momentum if self.reset_momentum else None,
                  a.int_arena if a.n_int > 0 else None, self.symm.peer_ptrs(o_int) if a.n_int > 0 else [],
                  self.loss_local, self.symm.peer_ptrs(o_loss), self.loss_out,
                  counts, from_flags, mask, self.rank, world, self.wire_kind, self.delta, nvls_now, self.epoch,
                  self.tile_flags, flag_value, tile, self.n_ctas, self.timeout_log2, self.status, self.phase_ns,
                  prepacked)
        with torch.cuda.stream(stream):
            if self.topk is not None:
                launch = self._C.fedavg_allreduce_topk
                own = (self.topk_rowptr_off, self.topk_off_off, self.topk_val_off)
            elif self.secagg is not None:
                launch = self._C.fedavg_allreduce_secagg
                self.secagg_sat.zero_()
                own = (self._secagg_words, self.secagg.range, self.secagg.frac_bits, self.secagg_sat)
            elif robust is not None and robust.kind == "krum":
                launch = self._C.fedavg_allreduce_krum
                own = (self.symm.peer_ptrs(o_clip), m, self.seg_stride,
                       self.symm.peer_ptrs(self.off_dist + par * self.half_dist), self.krum_work, self.krum_sync,
                       self.krum_report, *robust.krum_tables())
            elif robust is not None:
                launch = self._C.fedavg_allreduce_robust
                own = (self.symm.peer_ptrs(o_clip), m, self.seg_stride, robust.kind_id, robust.trim_table())
            elif self.local_range is not None:
                launch = self._C.fedavg_allreduce_local
                own = (self.local_range[0], self.local_range[1] - self.local_range[0])
            else:
                launch = self._C.fedavg_allreduce
                dp_args = ([], 0.0, 0, 0)
                if dp is not None:
                    from ..ops import functional as F
                    page = self.symm.view(o_clip, 1, torch.float32)
                    if clipped:
                        page.fill_(1.0)
                        self.dp_s.fill_(1.0)
                    else:     # theta is final here: the norm pass runs right before the collective, on its stream
                        F.dp_clip_factor(a.theta, a.global_w, dp.clip, self.dp_work, self.dp_s, self.dp_norm,
                                         s_copy_ptr=page.data_ptr(), nonfinite=self.dp_nonfinite)
                    seed = dp.seed - (1 << 64) if dp.seed >= (1 << 63) else dp.seed      # int64 bit pattern of the key
                    dp_args = (self.symm.peer_ptrs(o_clip), dp.noise_std, seed, self.dp_round())
                scaf_args = (None, None, 0, 0.0)
                if control is not None:
                    c, dc, n_clients = control
                    n_p = self.arena.n_param
                    scaf_args = (dc[:n_p], c[:n_p], self.seg1_off, 1.0 / float(n_clients))
                own = (*dp_args, *scaf_args)
            launch(*common, *own, *self._sopt_args())
        self.epoch = (self.epoch + 3) & 0xFFFFFFFF     # uint32 wrap: the kernel compares signed differences
        self.rounds += 1
        self._side_pending = on_side_stream

    def _sopt_args(self) -> tuple:
        """The collective's server-optimizer arguments ``(m, v, n_param, kind, coefficients)`` (``m`` None: off)."""
        if self.server_opt is None:
            return (None, None, 0, 0, [])
        a = self.arena
        return (a.server_m, a.server_v, a.n_param, self.server_opt.kind_id, self._sopt_coef)

    def server_state(self):
        """``(m, v)``: the server optimizer's state over the parameters (live tensors; ``v`` is None for FedAvgM)."""
        if self.server_opt is None:
            raise RuntimeError("server_state needs a session built with server_opt=")
        self.join()
        return self.arena.server_m, self.arena.server_v

    def last_secagg_saturation(self) -> int:
        """Elements this rank clamped to ``[-R, R]`` (or found non-finite) in the last secure round (a host read)."""
        if self.secagg is None:
            raise RuntimeError("last_secagg_saturation needs a session built with secagg=")
        self.join()
        return int(self.secagg_sat.item())

    def last_krum(self):
        """``(D, scores, kept)`` of the last Krum round, in segment order (a host read): the fp64 ``[P, P]`` squared
        distances the collective computed (non-finite: +inf), the fp64 ``[P]`` scores and the bool ``[P]`` kept mask.
        With ``P <= 2`` the collective skips the distances: ``D`` and the scores read 0 and the first ``m`` are kept."""
        if not self.krum:
            raise RuntimeError("last_krum needs a session built with robust=RobustConfig('krum', ...)")
        self.join()
        r = self.krum_report.cpu()
        mc = MAX_ROBUST_CLIENTS
        p = int(r[0])
        D = r[1: 1 + mc * mc].view(mc, mc)[:p, :p].clone()
        return D, r[1 + mc * mc: 1 + mc * mc + p].clone(), r[1 + mc * mc + mc: 1 + mc * mc + mc + p] != 0

    def dp_round(self) -> int:
        """Round index of the noise stream: ``(epoch - base_epoch) / 3``, identical on every rank (the plan's
        ``round`` in manager-driven rounds)."""
        return ((self.epoch - self.base_epoch) & 0xFFFFFFFF) // 3

    def last_clip_factors(self) -> List[float]:
        """This rank's clip factor of the last DP round (host read)."""
        return self.dp_s.tolist()

    def nonfinite_updates(self) -> int:
        """DP rounds so far in which this rank's update had a non-finite norm (and was given s = 0)."""
        return int(self.dp_nonfinite.item())

    def join(self) -> None:
        """Make the compute stream wait for a side-stream collective."""
        if getattr(self, "_side_pending", False):
            torch.cuda.current_stream(self.device).wait_stream(self.stream)
            self._side_pending = False

    def gate_first_layer(self, module, slot_name: Optional[str] = None) -> None:
        """bcast_gemm: make the NEXT forward of ``module`` (an ``ops.nn.Linear`` whose
        weight is the first GEMM operand of the model) wait, tile by tile, on the arrival
        flags this round's collective publishes, instead of on the whole kernel."""
        if self.tile_flags is None:
            raise RuntimeError("session was created with tile_flags=False")
        slot = None
        for name, s in self.arena.slots.items():
            if slot_name is not None and name == slot_name:
                slot = s
                break
            if slot_name is None and s.is_param and len(s.shape) == 2:
                owner = self.arena._owner(name)
                if owner is module:
                    slot = s
                    break
        if slot is None:
            raise ValueError("module weight not found in the arena")
        bias_off = -1
        if getattr(module, "bias", None) is not None:
            for name, s in self.arena.slots.items():
                if s.is_param and self.arena._owner(name) is module and name.endswith(".bias"):
                    bias_off = s.offset
        module.flags_cfg = {"flags": self.tile_flags, "epoch": self.rounds, "elem_off": slot.offset,
                            "tile_elems": self.FLAG_GRANULE, "bias_off": bias_off}

    def gate_first_conv(self, conv) -> None:
        """bcast_gemm for a convolutional first layer, usable INSIDE a captured CUDA graph: the staging kernel of the
        layer's weights and the TMA producer of its GEMM acquire the arrival flags of the arena granules under
        ``conv.weight`` and compare them with ``self.epoch_word`` -- a device word the session bumps (on the compute
        stream) every time it launches a collective.  Steps after the first of a round find the flags already there
        (one cached load), so every replay of the captured step can stay gated."""
        if self.tile_flags is None:
            raise RuntimeError("session was created with tile_flags=False")
        slot = None
        for name, s in self.arena.slots.items():
            if s.is_param and self.arena._owner(name) is conv and name.endswith(".weight"):
                slot = s
                break
        if slot is None:
            raise ValueError("conv weight not found in the arena")
        conv.flags_cfg = {"flags": self.tile_flags, "epoch_word": self.epoch_word, "elem_off": slot.offset,
                          "tile_elems": self.FLAG_GRANULE}

    def reduced_loss(self, n_epoch: int) -> List[float]:
        return self.loss_out[: min(n_epoch, MAX_LOSS)].tolist()

    def check(self) -> None:
        code = int(self.status.item())
        if code:
            self.status.zero_()
            raise RuntimeError("FedAvg collective timed out waiting for rank {}".format(code - 1))

    def _seg_bytes(self, n: int) -> int:
        if self.wire_kind == 2:
            return n + (n + 31) // 32
        return n * (2 if self.wire_kind == 1 else 4)

    def wire_bytes(self) -> int:
        """Bytes one client uploads per round (fp8: e4m3 payload + one UE8M0 scale byte per 32 elements); with
        SCAFFOLD, the model segment, its padding and the control-variate segment."""
        if self.scaffold:
            return self.seg1_off + self._seg_bytes(self.arena.n_param)
        return self._seg_bytes(self.n_wire)


class NcclSession:
    """Same contract through ``torch.distributed`` collectives (baseline / oracle)."""

    def __init__(self, arena: ParamArena, group=None, *, wire_dtype: str = "bf16", mode: str = "delta",
                 reset_momentum: bool = True, dp: Optional[DPConfig] = None, scaffold: bool = False,
                 robust: Optional[RobustConfig] = None, max_clients: int = 1, tile_flags: bool = False,
                 server_opt: Optional[ServerOptConfig] = None, topk: Optional[TopKConfig] = None,
                 local: bool = False, secagg: Optional[SecAggConfig] = None, **_unused):
        import torch.distributed as dist
        self._features = dict(wire_dtype=wire_dtype, mode=mode, scaffold=scaffold, topk=topk, server_opt=server_opt,
                             tile_flags=tile_flags, local=bool(local), secagg=secagg,
                              frozen=arena.frozen_range is not None)
        self.max_clients = _init_session(arena, self._features, dp, robust, max_clients)
        self.local_range = arena.skip_range
        self.topk, self.server_opt = topk, server_opt
        # top-k: k, this rank's upload of the round as a dense fp32 vector (zeros off its support) and its entry count
        self.topk_k = self.topk.k(n_float(arena)) if self.topk is not None else 0
        self._topk_up = None
        self._topk_entries = None
        self._topk_sent = None
        self.robust = robust
        self._last_krum = None
        self.scaffold = bool(scaffold)
        self.dist = dist
        self.arena, self.group, self.device = arena, group, arena.device
        self.dp = _agree_seed(dp, group)
        self.dp_s = [1.0]
        self.dp_nonfinite = 0
        self.wire_dtype = torch.bfloat16 if wire_dtype == "bf16" else torch.float32
        self.delta = mode == "delta"
        self.reset_momentum = reset_momentum
        inited = dist.is_available() and dist.is_initialized()
        self.world = dist.get_world_size(group) if inited else 1
        self.rank = dist.get_rank(group) if inited else 0
        self.wire = torch.zeros(arena.n_shared, dtype=self.wire_dtype, device=self.device)
        # robust: this rank's client segments (wire format) and how many of them pack_client filled this round
        self.segs = (torch.zeros(self.max_clients, arena.n, dtype=self.wire_dtype, device=self.device)
                     if robust is not None else None)
        self.counts = torch.zeros(self.world, dtype=torch.float32, device=self.device)
        self.secagg = secagg
        self._secagg_keys = _secagg_keys(secagg, group)
        self.secagg_saturated = 0
        self.loss_buf = torch.zeros(MAX_LOSS, dtype=torch.float32, device=self.device)
        self.loss_out = torch.zeros(MAX_LOSS, dtype=torch.float32, device=self.device)
        self.rounds = 0

    @torch.no_grad()
    def pack_client(self, j: int, reset: bool = False) -> None:
        """Segment ``j`` = the wire-format delta of the replica's client; ``reset`` returns the replica to the global
        model (as :meth:`FedAvgSession.pack_client`)."""
        if self.robust is None:
            raise RuntimeError("pack_client needs a session built with robust=")
        if not (0 <= int(j) < self.max_clients):
            raise ValueError("segment {} out of range (max_clients={})".format(j, self.max_clients))
        a = self.arena
        self.segs[int(j)].copy_((a.theta - a.global_w).to(self.wire_dtype))
        if reset:
            a.theta.copy_(a.global_w)
            a.sync_shadow()
            if a.momentum is not None:
                a.momentum.zero_()

    def _topk_residual(self, e: Optional[torch.Tensor]) -> Optional[torch.Tensor]:
        if self.topk is None:
            raise RuntimeError("top-k uploads need a session built with topk=")
        if not self.topk.error_feedback:
            return None
        if e is None or e.dtype != torch.float32 or e.numel() != self.arena.n:
            raise ValueError("error feedback needs the client's fp32 residual over the arena")
        return e

    @torch.no_grad()
    def pack_topk(self, e: Optional[torch.Tensor] = None) -> None:
        """This rank's upload = ``topk(u)`` of the replica's client, ``e`` updated (as :meth:`FedAvgSession.pack_topk`,
        through the host rule :func:`topk_ef_`)."""
        a = self.arena
        idx, vals = topk_ef_(a.theta, a.global_w, self._topk_residual(e), self.topk_k)
        self._topk_up = torch.zeros_like(a.theta)
        self._topk_up[idx] = vals
        self._topk_entries = int(idx.numel())

    @torch.no_grad()
    def fold_topk(self, acc: torch.Tensor, e: Optional[torch.Tensor], nk: float, first: bool, reset: bool) -> None:
        """``acc (+)= nk * topk(u)`` of the replica's client, ``e`` updated, and (``reset``) the replica reset."""
        a = self.arena
        idx, vals = topk_ef_(a.theta, a.global_w, self._topk_residual(e), self.topk_k)
        if first:
            acc.zero_()
        acc[idx] += vals * float(nk)
        if reset:
            a.theta.copy_(a.global_w)
            a.sync_shadow()
            if a.momentum is not None:
                a.momentum.zero_()

    @torch.no_grad()
    def pack_nonzero(self) -> None:
        """This rank's upload = ``theta - global`` (the folded mean of its clients), entries where they differ."""
        a = self.arena
        self._topk_up = a.theta - a.global_w
        self._topk_entries = int((a.theta != a.global_w).sum())

    def last_upload_entries(self) -> int:
        if self.topk is None:
            raise RuntimeError("last_upload_entries needs a session built with topk=")
        return self._topk_sent or 0

    def last_upload_bytes(self) -> int:
        if self.topk is None:
            return self.wire_bytes()
        if self._topk_sent is None:
            return 0
        return sparse_upload_bytes(self.arena.n, self._topk_sent,
                                   "bf16" if self.wire_dtype == torch.bfloat16 else "fp32")

    def _robust_update(self, counts, n_clients, robust: RobustConfig) -> torch.Tensor:
        """All-gather every rank's segments (padded to ``max_clients``) and their counts; ``robust_combine`` over the
        participants, rounded to the wire format as the fused kernel stores it."""
        a, dist = self.arena, self.dist
        if self.segs is None:       # a plain session asked for a robust round (seated plan): one segment
            self.segs = torch.zeros(1, a.n, dtype=self.wire_dtype, device=self.device)
        m = (1 if float(counts[self.rank]) != 0.0 else 0) if n_clients is None else int(n_clients)
        if not (0 <= m <= self.segs.shape[0]):
            raise ValueError("n_clients={} outside 0..max_clients={}".format(m, self.max_clients))
        if n_clients is None and m:
            self.segs[0].copy_((a.theta - a.global_w).to(self.wire_dtype))
        mine = self.segs.float()
        ms = torch.tensor([m], dtype=torch.int64, device=self.device)
        if self.world > 1:
            all_m = [torch.zeros_like(ms) for _ in range(self.world)]
            dist.all_gather(all_m, ms, group=self.group)
            all_s = [torch.zeros_like(mine) for _ in range(self.world)]
            dist.all_gather(all_s, mine, group=self.group)
        else:
            all_m, all_s = [ms], [mine]
        rows = [sg[: int(mk)] for sg, mk in zip(all_s, all_m)]
        stacked = torch.cat(rows, 0) if rows else mine[:0]
        if robust.kind == "krum":      # the same oracle, with the selection kept for last_krum()
            self._last_krum = krum_select(stacked, robust)
            stacked = stacked[self._last_krum[2].to(stacked.device)]
            robust = RobustConfig("trimmed_mean", 0.0)
        return robust_combine(stacked, robust).to(self.wire_dtype).float()

    def _secagg_update(self, counts: torch.Tensor, src: torch.Tensor) -> torch.Tensor:
        """The secure round's aggregate ``d``: this rank's masked upload (the encode kernel on CUDA, the numpy reference
        on the CPU; zeros when it does not participate), the int64 all-reduce of the uint32 words, the low 32 bits,
        decoded.  The nonce is the round counter."""
        cfg, f = self.secagg, self.secagg.frac_bits
        c = counts.tolist()
        w, _ = sa.weights(c)
        parts = [k for k, x in enumerate(c) if x > 0]
        nonce = (self.rounds & 0xFFFFFFFF, 0, 0)
        self.secagg_saturated = 0
        u = torch.zeros(src.numel(), dtype=torch.int64, device=self.device)
        if self.rank in parts:
            peers = sa.peer_list(self.rank, parts, self._secagg_keys)
            if src.is_cuda:
                from ..ops import functional as F
                out = torch.empty(src.numel(), dtype=torch.int32, device=self.device)
                sat = torch.zeros(1, dtype=torch.int64, device=self.device)
                F.secagg_encode(src.contiguous(), None, float(w[self.rank]), cfg.range, f, [k for k, _ in peers],
                                [s for _, s in peers], nonce, 0, out, sat)
                u = out.to(torch.int64) & 0xFFFFFFFF
                self.secagg_saturated = int(sat.item())
            else:
                q, self.secagg_saturated = sa.encode(src.numpy(), float(w[self.rank]), cfg.range, f)
                u = torch.from_numpy(sa.mask(q, peers, nonce).astype(np.int64))
        if self.world > 1:
            self.dist.all_reduce(u, group=self.group)
        u = u & 0xFFFFFFFF
        ring = torch.where(u >= 1 << 31, u - (1 << 32), u).to(torch.int32)     # int32(sum mod 2^32)
        return ring.float() * (2.0 ** -f)

    def last_secagg_saturation(self) -> int:
        """Elements this rank clamped (or found non-finite) in the last secure round."""
        if self.secagg is None:
            raise RuntimeError("last_secagg_saturation needs a session built with secagg=")
        return self.secagg_saturated

    def last_krum(self):
        """``(D, scores, kept)`` of the last Krum round in segment order, as :meth:`FedAvgSession.last_krum` (here the
        host oracle's fp64 values)."""
        if self._last_krum is None:
            raise RuntimeError("no Krum round has run on this session")
        return self._last_krum

    @torch.no_grad()
    def aggregate(self, n_samples_by_rank=None, alive_ranks=None, my_n=None, loss_history=None,
                  dp: Optional[DPConfig] = None, clipped: bool = False, round_index: Optional[int] = None,
                  control=None, n_clients: Optional[int] = None, robust: Optional[RobustConfig] = None,
                  **_unused) -> None:
        """DP-FedAvg (``dp``, default the session's): the same estimator as the fused kernel -- clip locally, all-reduce,
        then add the host-generated noise ``sigma C z(seed, round) / m`` after the reduce.  ``round_index`` (the
        manager's plan) sets the round counter, as it sets the fused session's barrier epoch.  ``control = (c, dc,
        n_clients)``: SCAFFOLD, as in :meth:`FedAvgSession.aggregate` -- all-reduce ``dc`` as a sum (a rank without
        participants contributes zeros), then ``c += sum / n_clients``."""
        dp = dp if dp is not None else self.dp
        robust = robust if robust is not None else self.robust
        if dp is not self.dp or robust is not self.robust:     # the session's own features were checked when built
            _session_rules(self._features, dp, robust)
        _check_control(self.scaffold, control)
        if round_index is not None:
            self.rounds = int(round_index)
        a, dist = self.arena, self.dist
        if n_samples_by_rank is not None:
            counts = torch.tensor([float(x) for x in n_samples_by_rank][: self.world], device=self.device)
        else:
            self.counts.zero_()
            self.counts[self.rank] = float(my_n)
            if self.world > 1:
                dist.all_reduce(self.counts, group=self.group)
            counts = self.counts
        total = counts.sum()
        w = counts[self.rank] / total
        # client-local entries: the round runs on the shared elements only, cat(x[:lo], x[hi:]), and writes them back
        theta, global_w = self._shared(a.theta), self._shared(a.global_w)
        src = (theta - global_w) if self.delta else theta
        if self.topk is not None:
            mine = float(counts[self.rank]) != 0.0
            if mine and self._topk_up is None:
                raise RuntimeError("a top-k round needs this rank's upload packed for it (pack_topk or pack_nonzero)")
            src = self._topk_up if mine else torch.zeros_like(a.theta)
            self._topk_sent = self._topk_entries if mine else None
            self._topk_up = None
        if robust is not None:
            upd = self._robust_update(counts, n_clients, robust)
            w = w if float(total) > 0.0 else torch.zeros_like(w)
        elif self.secagg is not None:
            upd = self._secagg_update(counts, src)
        elif n_clients is not None:
            raise ValueError("n_clients= needs a session built with robust=")
        elif dp is not None:
            s = 1.0
            if not clipped and float(counts[self.rank]) != 0.0:
                s, _ = clip_factor(src, dp.clip)
                self.dp_nonfinite += int(s == 0.0)
            self.dp_s = [s]
            wd = w * s
            if s == 0.0 or float(counts[self.rank]) == 0.0:
                src, wd = torch.zeros_like(src), 0.0          # a non-finite update contributes nothing (0 * nan = nan)
            self.wire.copy_((src * wd).to(self.wire_dtype))
        else:
            self.wire.copy_((src * w).to(self.wire_dtype))
        if self.world > 1 and robust is None and self.secagg is None:
            dist.all_reduce(self.wire, group=self.group)
        # every rank joins the loss reduce every round -- a rank that hosts no sampled client this round
        # contributes zeros (weight 0); skipping the call there would desynchronise the collectives
        self.loss_buf.zero_()
        if loss_history is not None:
            k = min(len(loss_history), MAX_LOSS)
            self.loss_buf[:k] = torch.tensor([float(x) for x in loss_history[:k]], device=self.device) * w
        if self.world > 1:
            dist.all_reduce(self.loss_buf, group=self.group)
        self.loss_out.copy_(self.loss_buf)
        d = None                        # the round's aggregate (delta mode)
        if robust is not None or self.secagg is not None:
            d = upd
        elif dp is not None and dp.noise_std > 0.0 and float(total) > 0.0:
            z = torch.from_numpy(normals(dp.seed, self.rounds & 0xFFFFFFFF, a.n)).to(device=self.device,
                                                                                      dtype=torch.float32)
            d = self.wire.float() + z * (dp.noise_std / float(total))
        elif self.delta:
            d = self.wire.float()
        if d is None:
            global_w.copy_(self.wire.float())
        elif self.server_opt is not None:
            if float(total) > 0.0:      # a round without weight leaves the model and the state unchanged
                n_p = a.n_param if self.local_range is None else self.local_range[0]   # the shared parameters
                apply_update_(global_w, d, n_p, a.server_m[:n_p], a.server_v[:n_p] if a.server_v is not None else None,
                              self.server_opt)
        else:
            global_w.add_(d)
        self._put(a.global_w, global_w)
        self._put(a.theta, global_w)
        if a.theta_bf16 is not None:
            self._put(a.theta_bf16, global_w.to(torch.bfloat16))
        if a.n_int > 0 and self.world > 1:
            dist.all_reduce(a.int_arena, op=dist.ReduceOp.MAX, group=self.group)
        if self.reset_momentum and a.momentum is not None:
            a.momentum[: self.local_range[0] if self.local_range is not None else a.momentum.numel()].zero_()
        if control is not None:
            c, dc, n_clients = control
            n_p = a.n_param
            tot = dc[:n_p].clone() if float(counts[self.rank]) != 0.0 else torch.zeros_like(c[:n_p])
            if self.world > 1:
                dist.all_reduce(tot, group=self.group)
            c[:n_p].add_(tot / float(n_clients))
        self.rounds += 1

    def _shared(self, x: torch.Tensor) -> torch.Tensor:
        """The elements the collective carries, as a new tensor: ``x`` without the client-local range."""
        if self.local_range is None:
            return x.clone()
        lo, hi = self.local_range
        return torch.cat((x[:lo], x[hi:]))

    def _put(self, dst: torch.Tensor, shared: torch.Tensor) -> None:
        """Write the shared elements back into ``dst`` around the client-local range."""
        if self.local_range is None:
            dst.copy_(shared)
            return
        lo, hi = self.local_range
        dst[:lo].copy_(shared[:lo])
        dst[hi:].copy_(shared[lo:])

    def dp_round(self) -> int:
        return self.rounds & 0xFFFFFFFF

    def server_state(self):
        """``(m, v)`` as :meth:`FedAvgSession.server_state`."""
        if self.server_opt is None:
            raise RuntimeError("server_state needs a session built with server_opt=")
        return self.arena.server_m, self.arena.server_v

    def last_clip_factors(self) -> List[float]:
        return list(self.dp_s)

    def nonfinite_updates(self) -> int:
        return self.dp_nonfinite

    def join(self) -> None:
        pass

    def reduced_loss(self, n_epoch: int) -> List[float]:
        return self.loss_out[: min(n_epoch, MAX_LOSS)].tolist()

    def check(self) -> None:
        pass

    def wire_bytes(self) -> int:
        n = self.arena.n_shared + (self.arena.n_param if self.scaffold else 0)
        return n * (2 if self.wire_dtype == torch.bfloat16 else 4)
