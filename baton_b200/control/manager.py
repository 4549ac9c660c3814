"""Parameter server: experiments, round orchestration, FedAvg aggregation.

Parity targets (reference file:line):
  * ``Manager``                        manager.py:10-18
  * ``Experiment``                     manager.py:21-132
  * ``trigger_start_round``            manager.py:51-64   GET /{name}/start_round?n_epoch=K
        default K = 32, 400 on a non-integer, 423 while a round is open,
        200 JSON {client_id: bool} ([] when there are no clients)
  * ``start_round``                    manager.py:70-93
  * ``update``                         manager.py:95-111  POST /{name}/update?client_id&key
        401 bad credentials, 410 {"error": "Wrong Update"} for a stale round
  * ``end_round`` (FedAvg)             manager.py:113-132
  * ``trigger_end_round`` / ``get_loss_history``   manager.py:66-68, 48-49

Fixed relative to the reference (SURVEY.md section 8): the two introspection
endpoints work (quirk 1), the zero-client round no longer leaks the lock
(quirk 2), a dead participant no longer wedges the round (quirk 14: eviction
drops it from the participant set and an optional ``round_timeout`` force-ends
the round).

New capabilities: client sampling (``sample_k`` / ``sample_fraction`` /
``?sample_k=``), pluggable data planes (``http`` | ``fused`` | ``nccl``),
checkpoint at ``end_round`` + resume, structured metrics (``/metrics``),
``/state``, and ``GET /{name}/evaluate`` (held-out loss and accuracy of the global
model, computed on the GPU seats of a seated data plane).
"""
from __future__ import annotations

import asyncio
import logging
import time
from typing import Any, List, Optional

from aiohttp import web

from .. import ckpt
from ..metrics import RoundMetrics
from ..parallel import wire
from ..parallel.aggregate import fedavg_loss_history
from ..parallel.dataplane import ManagerPlane, make_manager_plane
from ..parallel.dp import RDPAccountant
from ..utils.misc import SYSTEM_CLOCK, Clock, json_clean
from .client_manager import ClientManager
from .update_manager import UpdateException, UpdateManager

log = logging.getLogger("baton_b200.manager")

DEFAULT_N_EPOCH = 32  # manager.py:55


class Manager:
    """Container of experiments sharing one aiohttp application; every route is
    prefixed with ``/{experiment name}/`` so several jobs can coexist."""

    def __init__(self, app: web.Application, **experiment_defaults):
        self.app = app
        self.experiments: List["Experiment"] = []
        self.experiment_defaults = experiment_defaults

    def register_experiment(self, model, name: Optional[str] = None, **kwargs) -> "Experiment":
        name = name or getattr(model, "name", None) or hash(model)
        name = str(name)
        if any(e.name == name for e in self.experiments):
            raise ValueError("experiment {!r} already registered".format(name))
        opts = dict(self.experiment_defaults)
        opts.update(kwargs)
        experiment = Experiment(name, self.app, model, **opts)
        self.experiments.append(experiment)
        return experiment

    def __getitem__(self, name: str) -> "Experiment":
        for e in self.experiments:
            if e.name == name:
                return e
        raise KeyError(name)


class Experiment:
    def __init__(self, name: str, app: web.Application, model, client_ttl: float = 300, *,
                 dataplane: Any = "http", sample_k: Optional[int] = None,
                 sample_fraction: Optional[float] = None, seed: Optional[int] = None,
                 round_timeout: Optional[float] = None, checkpoint_dir: Optional[str] = None,
                 checkpoint_every: int = 1, resume: bool = False, clock: Clock = SYSTEM_CLOCK,
                 trusted_peers: bool = False, dp=None, dp_delta: float = 1e-5, robust=None):
        """``dp`` (a :class:`~baton_b200.parallel.dp.DPConfig`): aggregate with DP-FedAvg -- on the manager for the
        ``http`` plane, on the seats for the seated planes (the plan carries the clip norm, noise and key) -- and
        account every aggregated round at ``q`` = participants / registered clients; ``/metrics`` reports the
        ``(epsilon, dp_delta)`` spent.

        ``robust`` (a :class:`~baton_b200.parallel.robust.RobustConfig`): aggregate with the coordinate-wise median or
        trimmed mean of the participants' updates -- on the manager for the ``http`` plane, on the seats for the seated
        planes (the plan carries it); ``/metrics`` reports the aggregator."""
        self.name = name
        self.model = model
        self.app = app
        self.clock = clock
        self.client_manager = ClientManager(name, app, client_ttl, clock=clock, seed=seed)
        self.update_manager = UpdateManager(name)
        if robust is not None and dp is not None:
            raise ValueError("robust aggregation with DP-FedAvg is not supported")
        self.plane: ManagerPlane = make_manager_plane(dataplane, dp=dp, robust=robust)
        self.robust = robust
        self.dp = dp
        self.dp_delta = float(dp_delta)
        self.dp_accountant = RDPAccountant(dp.noise_multiplier) if dp is not None else None
        self._dp_q = 1.0
        self._dp_clipped = [0, 0]            # client updates with s < 1, client updates with a known factor
        self.sample_k = sample_k
        self.sample_fraction = sample_fraction
        self.round_timeout = round_timeout
        self.checkpoint_dir = checkpoint_dir
        self.checkpoint_every = max(1, int(checkpoint_every))
        self.trusted_peers = trusted_peers
        self.metrics = RoundMetrics(name)
        self.model_is_stale = False          # set by seated planes after a GPU-side reduce
        self.last_checkpoint: Optional[str] = None
        self._timeout_task: Optional[asyncio.Task] = None
        self._ending = False
        self._fanout_pending = False
        self._round_bytes = 0
        self.client_manager.add_evict_callback(self._on_client_evicted)
        self.register_handlers()
        if resume and checkpoint_dir:
            path = ckpt.latest_checkpoint(checkpoint_dir, name)
            if path:
                ckpt.load_checkpoint(path, self.model, self.update_manager)
                self.last_checkpoint = path
                log.info("resumed %s from %s (n_updates=%d)", name, path, self.update_manager.n_updates)
        app.on_cleanup.append(self._on_cleanup)

    # -- routes ------------------------------------------------------------
    def register_handlers(self) -> None:
        r = self.app.router
        r.add_post("/{}/update".format(self.name), self.update)
        r.add_get("/{}/start_round".format(self.name), self.trigger_start_round)
        r.add_get("/{}/end_round".format(self.name), self.trigger_end_round)
        r.add_get("/{}/loss_history".format(self.name), self.get_loss_history)
        r.add_get("/{}/state".format(self.name), self.get_state)
        r.add_get("/{}/metrics".format(self.name), self.get_metrics)
        r.add_get("/{}/state_dict".format(self.name), self.get_state_dict)
        r.add_get("/{}/evaluate".format(self.name), self.trigger_evaluate)

    async def _on_cleanup(self, app) -> None:
        self._cancel_timeout()

    # -- introspection -----------------------------------------------------
    async def get_loss_history(self, request: web.Request) -> web.Response:
        return web.json_response(list(self.update_manager.loss_history))

    async def get_state(self, request: web.Request) -> web.Response:
        return web.json_response(json_clean(self.update_manager.state()))

    async def get_metrics(self, request: web.Request) -> web.Response:
        out = self.metrics.summary()
        if self.dp is not None:
            out["dp"] = self.dp_summary()
        out["aggregator"] = self.robust.to_dict() if self.robust is not None else {"kind": "mean"}
        return web.json_response(json_clean(out))

    def dp_summary(self) -> dict:
        """Privacy spent so far: ``epsilon`` at ``delta`` over ``rounds`` aggregated DP rounds; ``clipped_fraction`` is
        the share of client updates with ``s < 1`` where the manager saw the factors (``http`` plane), else None."""
        eps, _ = self.dp_accountant.get_privacy_spent(self.dp_delta)
        known = self._dp_clipped[1]
        return {"clip": self.dp.clip, "noise_multiplier": self.dp.noise_multiplier,
                "rounds": self.dp_accountant.rounds, "epsilon": eps, "delta": self.dp_delta,
                "clipped_fraction": (self._dp_clipped[0] / known) if known else None}

    async def get_state_dict(self, request: web.Request) -> web.Response:
        """Pickled global ``state_dict`` (the checkpoint layout), refreshed from
        a data-plane seat first if a GPU-side reduce made the local copy stale."""
        await self.pull_global()
        body = wire.dumps({"state_dict": ckpt._cpu_state_dict(self.model),
                           "n_updates": self.update_manager.n_updates})
        return web.Response(body=body, content_type="application/octet-stream")

    # -- evaluation ----------------------------------------------------------
    async def trigger_evaluate(self, request: web.Request) -> web.Response:
        """Sample-weighted held-out loss and accuracy of the global model over the live seats that hold it.  Each seat
        evaluates its own held-out shard on its GPU (``POST /{name}/evaluate``); seats without held-out data answer
        501 and are left out.  423 while a round is open -- also when one opened or closed while the seats were
        evaluating, since they may then have evaluated different models (nothing is recorded) -- and 501 on the
        ``http`` plane (no seat holds the model)."""
        if self.plane.carries_tensors:
            return web.json_response({"err": "Evaluation needs a GPU-seated data plane"}, status=501)
        if self.update_manager.in_progress:
            return web.json_response({"err": "Update in progress"}, status=423)
        cm = self.client_manager
        n_updates = self.update_manager.n_updates
        seats = [cid for cid, rec in cm.clients.items() if rec.get("rank") is not None and rec.get("model_synced")]
        replies = await asyncio.gather(*(self._evaluate_seat(cid) for cid in seats))
        if self.update_manager.in_progress or self.update_manager.n_updates != n_updates:
            return web.json_response({"err": "Update in progress"}, status=423)
        got = [r for r in replies if r is not None]
        n = sum(r["n_samples"] for r in got)
        rec = self.metrics.add_eval(
            n_updates=self.update_manager.n_updates, n_seats=len(got), n_samples=n,
            loss=sum(r["loss_sum"] for r in got) / n if n else None,
            accuracy=sum(r["correct"] for r in got) / n if n else None)
        return web.json_response(json_clean(rec))

    async def _evaluate_seat(self, client_id: str) -> Optional[dict]:
        rec = self.client_manager.clients.get(client_id)
        if rec is None:
            return None
        url = "{}evaluate?client_id={}&key={}".format(rec["url"], client_id, rec["key"])
        try:
            async with self.client_manager._get_session().post(url) as resp:
                if resp.status != 200:
                    return None
                body = await resp.json()
        except Exception as exc:
            log.warning("evaluation on %s failed: %r", client_id, exc)
            return None
        try:
            out = {k: float(body[k]) for k in ("n_samples", "loss_sum", "correct")}
        except (KeyError, TypeError, ValueError):
            return None
        if any(v != v or v in (float("inf"), float("-inf")) for v in out.values()) or out["n_samples"] < 0:
            return None
        return out

    # -- round start -------------------------------------------------------
    async def trigger_start_round(self, request: web.Request) -> web.Response:
        try:
            n_epoch = int(request.query["n_epoch"])
        except KeyError:
            n_epoch = DEFAULT_N_EPOCH
        except ValueError:
            return web.json_response({"err": "Invalid Epoch Value"}, status=400)
        sample_k = None
        if "sample_k" in request.query:
            try:
                sample_k = int(request.query["sample_k"])
            except ValueError:
                return web.json_response({"err": "Invalid sample_k Value"}, status=400)
        try:
            status = await self.start_round(n_epoch, sample_k=sample_k)
        except UpdateException:
            return web.json_response({"err": "Update already in progress"}, status=423)
        return web.json_response(status)

    async def start_round(self, n_epoch: int, sample_k: Optional[int] = None,
                          extra: Optional[dict] = None):
        await self.update_manager.start_update(n_epoch=n_epoch)
        update_name = self.update_manager.update_name
        self._round_bytes = 0
        await self.client_manager.cull_clients()
        if not len(self.client_manager):
            log.info("no clients; aborting %s", update_name)
            self.update_manager.end_update()   # do not leak the round lock
            return []
        k = self.sample_k if sample_k is None else sample_k
        chosen = self.client_manager.sample(k, self.sample_fraction)
        self.update_manager.update_meta["sampled"] = list(chosen)
        self._dp_q = len(chosen) / float(len(self.client_manager))     # DP accounting: sampling rate of this round
        if self.plane.carries_tensors:
            await self.pull_global()
        body = self.plane.round_start_message(self.model, update_name, n_epoch, extra)
        self._round_bytes += len(body) * len(chosen)
        # seated planes: a seat that has never been given the global model (new, re-registered, or the manager resumed
        # a checkpoint) gets the full state_dict with this round_start; everybody else gets metadata only
        per_client = None
        need_model = self.plane.unsynced(self, chosen) if hasattr(self.plane, "unsynced") else []
        if need_model:
            await self.pull_global()
            full = self.plane.round_start_with_model(self.model, update_name, n_epoch, extra)
            self._round_bytes += (len(full) - len(body)) * len(need_model)
            need = set(need_model)
            per_client = lambda c: {"data": full} if c in need else {}      # noqa: E731
        async def _accepted(client_id: str, ok: bool) -> None:
            # a participant joins the round the moment ITS notify returns: a fast client may finish training and
            # POST its update while slower peers are still receiving the round (reference manager.py:87-89 only
            # registered participants after the whole gather)
            if ok and self.update_manager.in_progress and self.update_manager.update_name == update_name:
                self.update_manager.client_start(client_id)
            if ok and client_id in self.client_manager.clients and hasattr(self.plane, "unsynced"):
                self.client_manager.clients[client_id]["model_synced"] = True

        # while the fan-out is in flight the round cannot close on "everybody registered so far has reported": a fast seat
        # may train and report before a slower seat (e.g. one that is being sent the whole model) has even accepted
        self._fanout_pending = True
        try:
            result = await self.client_manager.notify_clients(
                "round_start", http_method="POST", data=body, clients=chosen, client_callback=_accepted,
                per_client_kwargs=per_client)
        finally:
            self._fanout_pending = False
        if not self.update_manager.in_progress or self.update_manager.update_name != update_name:
            return dict(result)          # every participant already reported and the round closed meanwhile
        if not self.update_manager:
            log.info("no clients working on %s; ending", update_name)
            await self.end_round()
        elif not self.update_manager.clients_left:
            await self.end_round()       # all updates arrived before the fan-out finished
        elif self.round_timeout:
            self._arm_timeout(update_name)
        return dict(result)

    # -- update ingestion --------------------------------------------------
    async def update(self, request: web.Request) -> web.Response:
        client_id = self.client_manager.verify_request(request)
        body = await request.read()
        try:
            data = wire.loads(body, trusted=self.trusted_peers)
        except Exception as exc:
            log.warning("undecodable update from %s: %r", client_id, exc)
            return web.json_response({"error": "Bad Payload"}, status=400)
        update_name = data.get("update_name")
        if (not self.update_manager.in_progress or
                update_name != self.update_manager.update_name):
            return web.json_response({"error": "Wrong Update"}, status=410)
        if client_id not in self.update_manager.clients:
            sampled = (self.update_manager.update_meta or {}).get("sampled") or ()
            if client_id not in sampled:
                # authenticated, right round, but never asked to take part in it
                return web.json_response({"error": "Wrong Update"}, status=410)
            # its round_start notify has not returned yet (we are still inside the fan-out): it did accept
            self.update_manager.client_start(client_id)
        problem = self._validate_update(data)
        if problem:
            log.warning("rejecting update from %s: %s", client_id, problem)
            return web.json_response({"error": "Bad Payload", "detail": problem}, status=400)
        self._round_bytes += len(body)
        self.update_manager.client_end(client_id, data)
        rec = self.client_manager[client_id]
        rec["last_update"] = update_name
        rec["num_updates"] += 1
        if not self.update_manager.clients_left and not self._fanout_pending:
            await self.end_round()       # (during the fan-out, start_round closes the round itself once it is complete)
        return web.json_response("OK")

    def _validate_update(self, data) -> Optional[str]:
        """Reason an update payload cannot be aggregated, or None.  A malformed upload is refused at the door
        (400) instead of poisoning ``end_round`` for everybody else."""
        if not isinstance(data, dict):
            return "payload is not a mapping"
        n = data.get("n_samples", 0)
        if isinstance(n, bool) or not isinstance(n, (int, float)) or n != n or n in (float("inf"), float("-inf")) or n < 0:
            return "n_samples must be a finite number >= 0"
        hist = data.get("loss_history", [])
        if not isinstance(hist, (list, tuple)) or any(
                isinstance(h, bool) or not isinstance(h, (int, float)) for h in hist):
            return "loss_history must be a list of numbers"
        if self.plane.carries_tensors and "state_dict" in data:
            sd = data["state_dict"]
            if not hasattr(sd, "keys"):
                return "state_dict is not a mapping"
            for key, ref in self.model.state_dict().items():
                if key not in sd:
                    return "state_dict is missing {!r}".format(key)
                val = sd[key]
                if not hasattr(val, "shape") or tuple(val.shape) != tuple(ref.shape):
                    return "state_dict[{!r}] has shape {} (expected {})".format(
                        key, tuple(getattr(val, "shape", ())), tuple(ref.shape))
                if ref.is_floating_point() != val.is_floating_point():
                    return "state_dict[{!r}] has dtype {} (expected {})".format(key, val.dtype, ref.dtype)
        return None

    # -- round end / aggregation --------------------------------------------
    async def trigger_end_round(self, request: web.Request) -> web.Response:
        await self.end_round()
        return web.json_response(json_clean(self.update_manager.state()))

    async def end_round(self) -> bool:
        """Close the open round and fold whatever arrived into the global model
        (sample-weighted mean over every ``state_dict`` entry, manager.py:119-126)
        and the loss history (manager.py:127-130)."""
        if not self.update_manager.in_progress or self._ending:
            return False
        self._ending = True
        try:
            self._cancel_timeout()
            update_name = self.update_manager.update_name
            meta = dict(self.update_manager.update_meta or {})
            n_participants = len(self.update_manager.clients)
            t0 = time.perf_counter()
            datas = dict(self.update_manager.client_responses)
            N = sum(d.get("n_samples", 0) for d in datas.values())
            aggregated = False
            try:
                if N:
                    # the collective runs while the round is still marked open so a
                    # concurrent /start_round gets 423 instead of racing the reduce
                    aggregated = await self.plane.aggregate(self, datas)
            except Exception:
                # a failed reduce must not wedge the experiment: the planes commit atomically, so the global
                # model is untouched; the round is closed (lock released) and reported as not aggregated
                log.exception("aggregation of %s failed; global model left unchanged", update_name)
                aggregated = False
            finally:
                self.update_manager.end_update()
            if aggregated and self.dp_accountant is not None:
                self.dp_accountant.step(self._dp_q)
                factors = getattr(self.plane, "last_clip_factors", None)
                if factors:
                    self._dp_clipped[0] += sum(1 for s in factors if s < 1.0)
                    self._dp_clipped[1] += len(factors)
            if not N:
                log.info("no responses for %s", update_name)
                self.metrics.add(update_name=update_name, n_clients=0, n_samples=0,
                                 participants=n_participants, aggregated=False,
                                 wall_s=self.update_manager.round_times[-1])
                return False
            ordered = list(datas.values())
            losses = fedavg_loss_history([d.get("loss_history", []) for d in ordered],
                                         [d.get("n_samples", 0) for d in ordered],
                                         meta.get("n_epoch"))
            self.update_manager.loss_history.extend(losses)
            rec = self.metrics.add(
                update_name=update_name, n_clients=len(datas), participants=n_participants,
                n_samples=int(N), n_epoch=meta.get("n_epoch"), aggregated=bool(aggregated),
                aggregate_s=time.perf_counter() - t0, bytes_http=self._round_bytes,
                plane=self.plane.name, wall_s=self.update_manager.round_times[-1],
                final_loss=losses[-1] if losses else None)
            if self.checkpoint_dir and self.update_manager.n_updates % self.checkpoint_every == 0:
                await self.save_checkpoint()
            log.info("finished %s final_loss=%s", update_name, rec["final_loss"])
            return True
        finally:
            self._ending = False

    # -- checkpoint / global model access ------------------------------------
    async def pull_global(self) -> bool:
        """Refresh ``self.model`` from a data-plane seat after a GPU-side
        reduce.  No-op for the http plane, whose reduce already wrote
        ``self.model``."""
        if not self.model_is_stale:
            return False
        cm = self.client_manager
        seats = sorted((rec.get("rank"), cid) for cid, rec in cm.clients.items()
                       if rec.get("rank") is not None)
        for _, cid in seats:
            rec = cm.clients.get(cid)
            if rec is None:
                continue
            url = "{}state_dict?client_id={}&key={}".format(rec["url"], cid, rec["key"])
            try:
                async with cm._get_session().get(url) as resp:
                    if resp.status != 200:
                        continue
                    body = await resp.read()
                sd = wire.loads(body, trusted=self.trusted_peers)["state_dict"]
                self.model.load_state_dict(sd)
                self.model_is_stale = False
                return True
            except Exception as exc:  # try the next seat
                log.warning("pull_global from %s failed: %r", cid, exc)
        return False

    async def save_checkpoint(self) -> Optional[str]:
        if not self.checkpoint_dir:
            return None
        await self.pull_global()
        loop = asyncio.get_running_loop()
        path = await loop.run_in_executor(
            None, lambda: ckpt.save_checkpoint(self.checkpoint_dir, self.name, self.model,
                                               self.update_manager))
        self.last_checkpoint = path
        return path

    # -- failure handling ------------------------------------------------------
    def _on_client_evicted(self, client_id: str, reason: str) -> None:
        if self.update_manager.client_drop(client_id):
            log.info("participant %s dropped from %s (%s)", client_id,
                     self.update_manager.update_name, reason)
            if self.update_manager.in_progress and not self.update_manager.clients_left and not self._fanout_pending:
                try:
                    asyncio.get_running_loop().create_task(self.end_round())
                except RuntimeError:  # no loop (sync test context)
                    pass

    def _arm_timeout(self, update_name: str) -> None:
        self._cancel_timeout()

        async def _expire():
            try:
                await asyncio.sleep(self.round_timeout)
            except asyncio.CancelledError:
                return
            if self.update_manager.in_progress and self.update_manager.update_name == update_name:
                log.warning("%s timed out after %.1fs; aggregating %d/%d", update_name,
                            self.round_timeout, len(self.update_manager.client_responses),
                            len(self.update_manager.clients))
                self._timeout_task = None
                await self.end_round()

        self._timeout_task = asyncio.ensure_future(_expire())

    def _cancel_timeout(self) -> None:
        task, self._timeout_task = self._timeout_task, None
        if task is not None and task is not asyncio.current_task():
            task.cancel()
