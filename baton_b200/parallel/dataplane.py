"""Tensor transport back-ends ("data planes") behind the control plane.

The reference has exactly one transport: pickled full ``state_dict`` in HTTP
bodies, star-shaped through the manager (manager.py:77-86, worker.py:108-118),
reduced afterwards on the manager CPU (manager.py:119-126).  Here that transport
is one of three interchangeable planes:

``http``   reference-compatible.  Tensors ride in the HTTP bodies, the manager
           reduces (CUDA weighted-sum kernel when its model lives on a GPU).
``fused``  one process per GPU on an NVSwitch box.  HTTP carries metadata only
           (``update_name``, ``n_samples``, ``loss_history``); parameters live in
           a symmetric flat arena and the end-of-round weighted reduce + global
           broadcast is ONE hand-written kernel doing peer loads / multicast
           stores over NVLink (``baton_b200.parallel.fedavg``).  The manager
           sends every seat the per-rank weight vector at ``end_round``.
``nccl``   the same metadata protocol with the reduce done by
           ``torch.distributed.all_reduce`` -- the baseline, and the test oracle.

Manager side and worker side are separate small classes because they run in
different processes.
"""
from __future__ import annotations

import logging
from typing import Any, Dict, List, Mapping, Optional

import torch

from . import wire
from .aggregate import dp_fedavg_into, fedavg_into, robust_into
from .features import check_features
from .server_opt import ServerOptConfig, server_step_

log = logging.getLogger("baton_b200.dataplane")


# ----------------------------------------------------------------------------
# manager side
# ----------------------------------------------------------------------------
class ManagerPlane:
    """What the parameter server needs from a transport."""

    name = "abstract"
    carries_tensors = True

    def round_start_message(self, model, update_name: str, n_epoch: int, extra: Optional[dict]) -> bytes:
        raise NotImplementedError

    def parse_update(self, body: bytes) -> dict:
        return wire.loads(body)

    async def aggregate(self, experiment, responses: Mapping[str, dict]) -> bool:
        raise NotImplementedError


class HttpManagerPlane(ManagerPlane):
    """Reference wire format: full weights in both directions.  ``dp`` (a :class:`~baton_b200.parallel.dp.DPConfig`):
    the manager aggregates with DP-FedAvg (:func:`~baton_b200.parallel.aggregate.dp_fedavg_into`) instead of the
    sample-weighted mean.  As in the plain mean, an upload with ``n_samples == 0`` (a client that trained nothing) is
    not a participant; a round without participants aggregates nothing and does not advance the noise stream.
    ``last_clip_factors`` holds the factors of the last aggregated round.  ``robust`` (a
    :class:`~baton_b200.parallel.robust.RobustConfig`, exclusive with ``dp``): the coordinate-wise median / trimmed mean
    or the Multi-Krum mean of the participants' updates (:func:`~baton_b200.parallel.aggregate.robust_into`), uploads
    with ``n_samples == 0`` excluded as under DP.  ``server_opt`` (a
    :class:`~baton_b200.parallel.server_opt.ServerOptConfig`): the round's aggregate is computed as above into a scratch
    copy, then ``d = scratch - live`` over the model's parameters (``named_parameters`` order, one fp32 vector) drives
    :func:`~baton_b200.parallel.server_opt.server_step_`; buffers take the aggregate as before.  The state ``(m, v)``
    lives here (:meth:`server_state`, :meth:`load_server_state`)."""

    name = "http"
    carries_tensors = True

    def __init__(self, int_policy: str = "max", dp=None, robust=None, server_opt=None):
        check_features(dp=dp, robust=robust, server_opt=server_opt, plane="http")
        if server_opt is not None and not isinstance(server_opt, ServerOptConfig):
            raise TypeError("server_opt= takes a ServerOptConfig")
        self.int_policy = int_policy
        self.dp = dp
        self.robust = robust
        self.server_opt = server_opt
        self.server_m: Optional[torch.Tensor] = None     # allocated by the first server step (m = 0, v = tau^2)
        self.server_v: Optional[torch.Tensor] = None
        self.dp_rounds = 0
        self.last_clip_factors: List[float] = []

    def round_start_message(self, model, update_name, n_epoch, extra=None) -> bytes:
        sd = model.state_dict()
        # detach+cpu so CUDA-resident global models still produce a payload a
        # CPU-only worker can load (the reference is CPU-only throughout)
        sd = type(sd)((k, v.detach().to("cpu")) for k, v in sd.items())
        msg = {"state_dict": sd, "update_name": update_name, "n_epoch": n_epoch}
        if extra:
            msg.update(extra)
        return wire.dumps(msg)

    async def aggregate(self, experiment, responses) -> bool:
        datas = [d for d in responses.values() if "state_dict" in d]
        if not datas:
            return False
        # reduce into a scratch copy and commit only when every key went through: a client payload that makes
        # the reduce raise half-way must not leave the global model half-written
        live = experiment.model.state_dict()
        scratch = type(live)((k, v.detach().clone()) for k, v in live.items())
        if self.robust is not None:
            datas = [d for d in datas if float(d.get("n_samples", 0)) > 0]
            ok = robust_into(scratch, [d["state_dict"] for d in datas], self.robust, int_policy=self.int_policy)
        elif self.dp is not None:
            datas = [d for d in datas if float(d.get("n_samples", 0)) > 0]
            if not datas:
                return False
            self.last_clip_factors = dp_fedavg_into(scratch, [d["state_dict"] for d in datas], clip=self.dp.clip,
                                                    noise_multiplier=self.dp.noise_multiplier, seed=self.dp.seed,
                                                    round_index=self.dp_rounds, int_policy=self.int_policy)
            self.dp_rounds += 1
            ok = True
        else:
            ok = fedavg_into(scratch, [d["state_dict"] for d in datas], [d["n_samples"] for d in datas],
                             int_policy=self.int_policy)
        if ok and self.server_opt is not None:
            self._server_step(experiment.model, live, scratch)
        if ok:
            with torch.no_grad():
                for k, v in live.items():
                    v.copy_(scratch[k])
        return ok

    @torch.no_grad()
    def _server_step(self, model, live, scratch) -> None:
        """Replace the parameters' aggregate in ``scratch`` by the server optimizer's step from ``live``."""
        names = [n for n, _ in model.named_parameters()]
        x = torch.cat([live[n].detach().reshape(-1).float() for n in names])
        d = torch.cat([scratch[n].reshape(-1).float() for n in names]) - x
        if self.server_m is None or self.server_m.numel() != x.numel():
            self.server_m, self.server_v = self.server_opt.init_state(x.numel(), x.device)
        server_step_(x, d, self.server_m, self.server_v, self.server_opt)
        off = 0
        for n in names:
            t = scratch[n]
            t.copy_(x[off: off + t.numel()].view(t.shape).to(t.dtype))
            off += t.numel()

    def server_state(self) -> Optional[dict]:
        """The checkpoint entry of the server optimizer: ``{"config", "m", "v"}`` on the CPU (``m`` / ``v`` None before
        the first step, ``v`` None for FedAvgM), or None without one."""
        if self.server_opt is None:
            return None
        cpu = (lambda t: t.detach().to("cpu").clone() if t is not None else None)
        return {"config": self.server_opt.to_dict(), "m": cpu(self.server_m), "v": cpu(self.server_v)}

    def load_server_state(self, entry: Optional[dict], device=None) -> None:
        """Restore :meth:`server_state`; ``None`` (a checkpoint without the entry) restores the initial state."""
        if self.server_opt is None:
            return
        if entry is None or entry.get("m") is None:
            self.server_m = self.server_v = None
            return
        saved = ServerOptConfig.from_dict(entry["config"])
        if saved != self.server_opt:
            raise ValueError("the checkpoint's server optimizer {} differs from this experiment's {}".format(
                saved.to_dict(), self.server_opt.to_dict()))
        self.server_m = entry["m"].to(device=device, dtype=torch.float32)
        self.server_v = entry["v"].to(device=device, dtype=torch.float32) if entry.get("v") is not None else None


class SeatedManagerPlane(ManagerPlane):
    """Metadata-only plane for clients seated on a GPU data plane (``fused`` or
    ``nccl``).  ``aggregate`` turns the round's ``n_samples`` into a per-rank
    weight vector and POSTs it to every live seat; the seats run the collective
    kernel together.  The manager's own ``model`` is refreshed lazily through
    ``Experiment.pull_global``.

    The manager stays the authority for two things the seats cannot agree on by themselves:

    * the MODEL: a seat that has not been given the global model yet (first round after it registered -- including
      a re-registration after an eviction -- or after the manager resumed from a checkpoint) receives the full
      ``state_dict`` inside its ``round_start`` (reference behaviour, manager.py:77-86); synced seats get metadata only;
    * the ROUND INDEX of the collective: every plan carries ``round`` = aggregations dispatched so far, from which
      every seat derives the same barrier epoch, so a seat that sat out rounds re-enters in step with its peers."""

    carries_tensors = False

    def __init__(self, name: str = "fused", world_size: Optional[int] = None, distribute_initial: bool = True,
                 dp=None, robust=None):
        check_features(dp=dp, robust=robust, plane="seated")
        # robust (a RobustConfig): the plan carries {"robust": RobustConfig.to_dict()}; every seat uploads one segment
        self.robust = robust
        self.name = name
        self.world_size = world_size
        self.distribute_initial = distribute_initial
        self.n_aggregates = 0
        # DP-FedAvg (a DPConfig): the plan weights count CLIENTS per rank and carries {"dp": {clip, noise_multiplier,
        # seed}}, so every seat runs the same estimator with the manager's noise key
        self.dp = dp

    def round_start_message(self, model, update_name, n_epoch, extra=None) -> bytes:
        msg = {"update_name": update_name, "n_epoch": n_epoch, "dataplane": self.name}
        if extra:
            msg.update(extra)
        return wire.dumps(msg, prefer_json=True)

    def unsynced(self, experiment, chosen) -> List[str]:
        """Clients of this round that still need the global model."""
        if not self.distribute_initial:
            return []
        cm = experiment.client_manager
        return [c for c in chosen if c in cm.clients and not cm.clients[c].get("model_synced")]

    def round_start_with_model(self, model, update_name, n_epoch, extra=None) -> bytes:
        sd = model.state_dict()
        sd = type(sd)((k, v.detach().to("cpu")) for k, v in sd.items())
        msg = {"state_dict": sd, "update_name": update_name, "n_epoch": n_epoch, "dataplane": self.name}
        if extra:
            msg.update(extra)
        return wire.dumps(msg)

    def rank_weights(self, experiment, responses) -> Dict[str, Any]:
        cm = experiment.client_manager
        seats: Dict[int, float] = {}
        alive: List[int] = []
        for cid, rec in cm.clients.items():
            if rec.get("rank") is not None:
                alive.append(int(rec["rank"]))
        for cid, d in responses.items():
            rec = cm.clients.get(cid)
            rank = d.get("rank", rec.get("rank") if rec else None)
            if rank is None:
                continue
            n = float(d["n_samples"])
            if self.dp is not None:
                n = 1.0 if n > 0 else 0.0          # DP: uniform over the clients that trained
            seats[int(rank)] = seats.get(int(rank), 0.0) + n
        world = self.world_size or (max(alive + list(seats)) + 1 if (alive or seats) else 0)
        n_by_rank = [seats.get(r, 0.0) for r in range(world)]
        plan = {"n_samples_by_rank": n_by_rank, "alive_ranks": sorted(set(alive) | set(seats))}
        if self.dp is not None:
            plan["dp"] = {"clip": self.dp.clip, "noise_multiplier": self.dp.noise_multiplier, "seed": self.dp.seed}
        if self.robust is not None:
            plan["robust"] = self.robust.to_dict()
        return plan

    async def aggregate(self, experiment, responses) -> bool:
        plan = self.rank_weights(experiment, responses)
        if sum(plan["n_samples_by_rank"]) <= 0:
            return False
        plan["update_name"] = experiment.update_manager.update_name
        plan["round"] = self.n_aggregates           # seats derive the collective's barrier epoch from it
        body = wire.dumps(plan, prefer_json=True)
        cm = experiment.client_manager
        seats = [cid for cid, rec in cm.clients.items() if rec.get("rank") is not None]
        self.n_aggregates += 1          # the epoch advances whether or not every seat answers
        result = await cm.notify_clients("aggregate", http_method="POST", data=body, clients=seats)
        ok = [cid for cid, r in result if r]
        log.info("aggregate dispatched to %d/%d seats", len(ok), len(seats))
        experiment.model_is_stale = True
        return bool(ok)


# ----------------------------------------------------------------------------
# worker side
# ----------------------------------------------------------------------------
class WorkerPlane:
    name = "abstract"
    carries_tensors = True
    rank: Optional[int] = None

    def registration_extras(self) -> dict:
        return {}

    def receive_round(self, worker, msg: dict) -> None:
        raise NotImplementedError

    def update_message(self, worker, update_name, n_samples, loss_history) -> bytes:
        raise NotImplementedError

    def aggregate(self, worker, plan: dict) -> None:
        raise NotImplementedError("this data plane aggregates on the manager")

    def export_state(self, worker) -> bytes:
        sd = worker.model.state_dict()
        sd = type(sd)((k, v.detach().to("cpu")) for k, v in sd.items())
        return wire.dumps({"state_dict": sd})


class HttpWorkerPlane(WorkerPlane):
    name = "http"

    def receive_round(self, worker, msg) -> None:
        worker.model.load_state_dict(msg["state_dict"])

    def update_message(self, worker, update_name, n_samples, loss_history) -> bytes:
        sd = worker.model.state_dict()
        sd = type(sd)((k, v.detach().to("cpu")) for k, v in sd.items())
        return wire.dumps({"state_dict": sd, "n_samples": n_samples,
                           "update_name": update_name, "loss_history": list(loss_history)})


class SeatedWorkerPlane(WorkerPlane):
    """Worker half of the ``fused`` / ``nccl`` planes.  ``session`` is a
    :class:`baton_b200.parallel.fedavg.FedAvgSession` (or any object with
    ``rank``, ``aggregate(n_samples_by_rank, alive_ranks)``)."""

    carries_tensors = False

    def __init__(self, session, name: str = "fused"):
        self.session = session
        self.name = name
        self.rank = int(session.rank)

    def registration_extras(self) -> dict:
        return {"rank": self.rank, "backend": self.name,
                "device": str(getattr(self.session, "device", "cpu"))}

    def receive_round(self, worker, msg) -> None:
        # normally the weights are already resident: the previous round's fused reduce wrote the new global model
        # straight into this replica's arena (the reference's load_state_dict, worker.py:98, has nothing left to do).
        # The manager attaches the state_dict when this seat is new / rejoining / the manager resumed a checkpoint.
        if "state_dict" in msg:
            worker.model.load_state_dict(msg["state_dict"])
            arena = getattr(worker, "arena", None) or getattr(self.session, "arena", None)
            if arena is not None:
                arena.commit_global()       # these weights ARE the global model: refresh global_w + bf16 shadow
            if hasattr(self.session, "stale"):
                self.session.stale = False

    def update_message(self, worker, update_name, n_samples, loss_history) -> bytes:
        return wire.dumps({"n_samples": n_samples, "update_name": update_name,
                           "loss_history": [float(x) for x in loss_history],
                           "rank": self.rank, "dataplane": self.name}, prefer_json=True)

    def aggregate(self, worker, plan) -> None:
        kw = {}
        # the round index sets the barrier epoch of the fused session and, under DP, the noise stream's round
        if plan.get("round") is not None and (hasattr(self.session, "base_epoch") or plan.get("dp")):
            kw["round_index"] = int(plan["round"])
        if plan.get("dp"):
            from .dp import DPConfig
            d = plan["dp"]
            kw["dp"] = DPConfig(float(d["clip"]), float(d["noise_multiplier"]), seed=int(d["seed"]))
        if plan.get("robust"):
            from .robust import RobustConfig
            kw["robust"] = RobustConfig.from_dict(plan["robust"])
        self.session.aggregate(plan["n_samples_by_rank"], plan.get("alive_ranks"), **kw)
        check = getattr(self.session, "check", None)
        if check is not None:
            check()             # a peer that died mid-collective surfaces here as an error, not as a hang


def make_manager_plane(spec, dp=None, robust=None, server_opt=None) -> ManagerPlane:
    http = spec in (None, "http", "http_pickle") or isinstance(spec, HttpManagerPlane)
    check_features(dp=dp, robust=robust, server_opt=server_opt, plane="http" if http else "seated")
    if isinstance(spec, ManagerPlane):
        if server_opt is not None and getattr(spec, "server_opt", None) != server_opt:
            raise ValueError("a server-optimizer experiment needs a data plane built with the same server_opt=")
        if dp is not None and getattr(spec, "dp", None) is None:
            raise ValueError("a DP experiment needs a data plane built with the same dp=")
        if robust is not None and getattr(spec, "robust", None) is None:
            raise ValueError("a robust experiment needs a data plane built with the same robust=")
        return spec
    if http:
        return HttpManagerPlane(dp=dp, robust=robust, server_opt=server_opt)
    if spec in ("fused", "nccl"):
        return SeatedManagerPlane(spec, dp=dp, robust=robust)
    raise ValueError("unknown data plane {!r}".format(spec))


def make_worker_plane(spec, session=None) -> WorkerPlane:
    if isinstance(spec, WorkerPlane):
        return spec
    if spec in (None, "http", "http_pickle"):
        return HttpWorkerPlane()
    if spec in ("fused", "nccl"):
        if session is None:
            raise ValueError("the {!r} plane needs a FedAvgSession".format(spec))
        return SeatedWorkerPlane(session, spec)
    raise ValueError("unknown data plane {!r}".format(spec))
