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
"""
from __future__ import annotations

from typing import List, Optional, Sequence

import torch

from .arena import ParamArena
from .dp import DPConfig, clip_factor, normals
from .robust import MAX_ROBUST_CLIENTS, RobustConfig, robust_combine
from .symm import SymmetricBuffer

MAX_LOSS = 64       # per-epoch loss slots carried through the collective
MAX_CTAS = 296      # pad slots; the kernel runs one 512-thread CTA per SM (132 on H100 SXM), clamped by the launcher


def _align(x: int, a: int) -> int:
    return (x + a - 1) // a * a


def _check_dp_mode(dp: Optional[DPConfig], delta: bool) -> None:
    if dp is not None and not delta:
        raise ValueError("DP-FedAvg clips and noises the update theta - global: it needs mode='delta'")


def _check_scaffold(scaffold: bool, dp: Optional[DPConfig], delta: bool) -> None:
    if scaffold and not delta:
        raise ValueError("SCAFFOLD needs mode='delta'")
    if scaffold and dp is not None:
        raise ValueError("SCAFFOLD and DP-FedAvg are exclusive: DP would have to clip and noise dc too")


def _check_robust(robust: Optional[RobustConfig], dp: Optional[DPConfig], scaffold: bool, delta: bool,
                  tile_flags: bool, max_clients: int) -> int:
    if robust is None:
        if int(max_clients) != 1:
            raise ValueError("max_clients > 1 needs a robust aggregator: plain rounds fold their clients into one upload")
        return 1
    if not isinstance(robust, RobustConfig):
        raise TypeError("robust= takes a RobustConfig")
    if not delta:
        raise ValueError("robust aggregation combines the updates theta - global: it needs mode='delta'")
    if dp is not None:
        raise ValueError("robust aggregation with DP-FedAvg is not supported: DP's sensitivity bound assumes the clipped "
                         "mean")
    if scaffold:
        raise ValueError("robust aggregation with SCAFFOLD is not supported: its control-variate update is a mean")
    if tile_flags:
        raise ValueError("robust aggregation with tile_flags is not supported")
    if not (1 <= int(max_clients) <= MAX_ROBUST_CLIENTS):
        raise ValueError("max_clients must be in 1..{}, got {!r}".format(MAX_ROBUST_CLIENTS, max_clients))
    return int(max_clients)


def _check_control(scaffold: bool, control) -> None:
    if scaffold and control is None:
        raise ValueError("a SCAFFOLD session needs control=(c, dc, n_clients) every round")
    if not scaffold and control is not None:
        raise ValueError("control= needs a session built with scaffold=True")


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
                 scaffold: bool = False, robust: Optional[RobustConfig] = None, max_clients: int = 1):
        from ..ops._ext import load
        self._C = load()
        assert wire_dtype in ("bf16", "fp32", "fp8") and mode in ("delta", "weights")
        _check_dp_mode(dp, mode == "delta")
        _check_scaffold(scaffold, dp, mode == "delta")
        self.max_clients = _check_robust(robust, dp, scaffold, mode == "delta", tile_flags, max_clients)
        self.robust = robust
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
        self.half_wire = _align(half, 2 << 20)                        # multicast-friendly granularity
        self.half_int = _align(max(arena.n_int, 1) * 8, 256)
        self.half_loss = _align(MAX_LOSS * 4, 256)
        self.half_clip = 256                                          # DP: this rank's clip factor s_r; robust: m_r
        self.off_wire = 0
        self.off_int = 2 * self.half_wire
        self.off_loss = self.off_int + 2 * self.half_int
        self.off_clip = self.off_loss + 2 * self.half_loss
        self.off_pads = _align(self.off_clip + 2 * self.half_clip, 256)
        total = _align(self.off_pads + (MAX_CTAS + 8) * self._C.MAX_RANKS * 8, 2 << 20)
        self.symm = SymmetricBuffer(total, self.device, group)
        self.rank, self.world = self.symm.rank, self.symm.world
        assert self.world <= self._C.MAX_RANKS
        self.use_nvls = self.symm.has_multicast if nvls == "auto" else (bool(nvls) and self.symm.has_multicast)
        if self.wire_kind == 2:
            self.use_nvls = False      # the switch adds raw elements; block scales need the P2P path
        self.dp = _agree_seed(dp, group)
        if self.dp is not None or self.scaffold or self.robust is not None:
            # the clip factors / the 1 / N of the control variates are applied by the readers, and a selection is not
            # a sum: peer loads only
            self.use_nvls = False
        self._packed_epoch = None   # robust: barrier epoch whose wire half pack_client filled
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
        t = torch.tensor([best[False], best[True]], device=self.device, dtype=torch.float64)
        dist.all_reduce(t, op=dist.ReduceOp.MAX, group=self.group)
        self.use_nvls = bool(t[1] < t[0])
        self.nvls_choice = "autotuned p2p {:.0f} us vs nvls {:.0f} us".format(float(t[0]) * 1e3, float(t[1]) * 1e3)
        self.check()
        self.symm.barrier()

    # ------------------------------------------------------------------ K4: upload copy emitted by the optimizer
    def pack_spec(self) -> Optional[dict]:
        """Arguments for ``ops.fused_sgd(pack=...)`` (stable device tensors: safe to capture), or None when the wire
        format needs the in-kernel pack (block-scaled fp8)."""
        if self.wire_kind == 2 or self.device.type != "cuda":
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
        _check_dp_mode(dp, self.delta)
        _check_control(self.scaffold, control)
        if control is not None and dp is not None:
            raise ValueError("SCAFFOLD and DP-FedAvg are exclusive")
        robust = robust if robust is not None else self.robust
        if robust is not None and robust is not self.robust:
            _check_robust(robust, dp, self.scaffold, self.delta, self.tile_flags is not None, 1)
        if robust is None and n_clients is not None:
            raise ValueError("n_clients= needs a robust session or robust=")
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
        nvls_now = bool(self.use_nvls and len(alive) == world and dp is None and robust is None)
        want_scale = (counts[self.rank] if not from_flags else float(my_n)) if (self.use_nvls and world > 1) else 1.0
        prepacked = bool(prepacked and self.wire_kind != 2 and self._armed_for == (self.epoch, float(want_scale))
                         and (nvls_now == bool(self.use_nvls and world > 1)))
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
            per = -(-a.n // (len(alive) * self.n_ctas))
            tile = max(self.min_tile, (per + 31) // 32 * 32)
        if self.tile_flags is not None:      # arrival flags cover fixed 1024-element granules: tiles must not split one
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
        if robust is not None:
            with torch.cuda.stream(stream):
                self._C.fedavg_allreduce_robust(
                    self.symm.peer_ptrs(o_wire), self.symm.peer_ptrs(self.off_pads),
                    a.theta, a.global_w, a.theta_bf16, a.momentum if self.reset_momentum else None,
                    a.int_arena if a.n_int > 0 else None, self.symm.peer_ptrs(o_int) if a.n_int > 0 else [],
                    self.loss_local, self.symm.peer_ptrs(o_loss), self.loss_out,
                    counts, from_flags, mask, self.rank, world, self.wire_kind, self.epoch, tile, self.n_ctas,
                    self.timeout_log2, self.status, self.phase_ns, prepacked,
                    self.symm.peer_ptrs(o_clip), m, self.seg_stride, robust.kind_id, robust.trim_table())
            self.epoch = (self.epoch + 3) & 0xFFFFFFFF
            self.rounds += 1
            self._side_pending = on_side_stream
            return
        with torch.cuda.stream(stream):
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
            self._C.fedavg_allreduce(
                self.symm.peer_ptrs(o_wire), self.symm.peer_ptrs(self.off_pads),
                self.symm.mc(o_wire) if nvls_now else 0,
                a.theta, a.global_w, a.theta_bf16,
                a.momentum if self.reset_momentum else None,
                a.int_arena if a.n_int > 0 else None,
                self.symm.peer_ptrs(o_int) if a.n_int > 0 else [],
                self.loss_local, self.symm.peer_ptrs(o_loss), self.loss_out,
                counts, from_flags, mask, self.rank, world, self.wire_kind, self.delta,
                nvls_now, self.epoch,
                self.tile_flags, flag_value, tile, self.n_ctas, self.timeout_log2, self.status, self.phase_ns,
                prepacked, *dp_args, *scaf_args)
        self.epoch = (self.epoch + 3) & 0xFFFFFFFF     # uint32 wrap: the kernel compares signed differences
        self.rounds += 1
        self._side_pending = on_side_stream

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
        return self._seg_bytes(self.arena.n)


class NcclSession:
    """Same contract through ``torch.distributed`` collectives (baseline / oracle)."""

    def __init__(self, arena: ParamArena, group=None, *, wire_dtype: str = "bf16", mode: str = "delta",
                 reset_momentum: bool = True, dp: Optional[DPConfig] = None, scaffold: bool = False,
                 robust: Optional[RobustConfig] = None, max_clients: int = 1, tile_flags: bool = False, **_unused):
        import torch.distributed as dist
        _check_dp_mode(dp, mode == "delta")
        _check_scaffold(scaffold, dp, mode == "delta")
        self.max_clients = _check_robust(robust, dp, scaffold, mode == "delta", tile_flags, max_clients)
        self.robust = robust
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
        self.wire = torch.zeros(arena.n, dtype=self.wire_dtype, device=self.device)
        # robust: this rank's client segments (wire format) and how many of them pack_client filled this round
        self.segs = (torch.zeros(self.max_clients, arena.n, dtype=self.wire_dtype, device=self.device)
                     if robust is not None else None)
        self.counts = torch.zeros(self.world, dtype=torch.float32, device=self.device)
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
        return robust_combine(stacked, robust).to(self.wire_dtype).float()

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
        _check_control(self.scaffold, control)
        if round_index is not None:
            self.rounds = int(round_index)
        a, dist = self.arena, self.dist
        dp = dp if dp is not None else self.dp
        _check_dp_mode(dp, self.delta)
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
        src = (a.theta - a.global_w) if self.delta else a.theta
        robust = robust if robust is not None else self.robust
        if robust is not None:
            upd = self._robust_update(counts, n_clients, robust)
            w = w if float(total) > 0.0 else torch.zeros_like(w)
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
        if self.world > 1 and robust is None:
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
        if robust is not None:
            a.global_w.add_(upd)
        elif dp is not None and dp.noise_std > 0.0 and float(total) > 0.0:
            z = torch.from_numpy(normals(dp.seed, self.rounds & 0xFFFFFFFF, a.n)).to(device=self.device,
                                                                                      dtype=torch.float32)
            a.global_w.add_(self.wire.float() + z * (dp.noise_std / float(total)))
        elif self.delta:
            a.global_w.add_(self.wire.float())
        else:
            a.global_w.copy_(self.wire.float())
        a.theta.copy_(a.global_w)
        if a.theta_bf16 is not None:
            a.theta_bf16.copy_(a.theta.to(torch.bfloat16))
        if a.n_int > 0 and self.world > 1:
            dist.all_reduce(a.int_arena, op=dist.ReduceOp.MAX, group=self.group)
        if self.reset_momentum and a.momentum is not None:
            a.momentum.zero_()
        if control is not None:
            c, dc, n_clients = control
            n_p = a.n_param
            tot = dc[:n_p].clone() if float(counts[self.rank]) != 0.0 else torch.zeros_like(c[:n_p])
            if self.world > 1:
                dist.all_reduce(tot, group=self.group)
            c[:n_p].add_(tot / float(n_clients))
        self.rounds += 1

    def dp_round(self) -> int:
        return self.rounds & 0xFFFFFFFF

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
        n = self.arena.n + (self.arena.n_param if self.scaffold else 0)
        return n * (2 if self.wire_dtype == torch.bfloat16 else 4)
