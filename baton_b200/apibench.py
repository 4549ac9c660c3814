"""``bench.py --api http``: the flagship round driven through Baton's own API on N GPUs.

Topology (what a user of the reference runs, reference demo.py:62-77, on the NVLink data plane):

    manager process (CPU)   ``python demo.py manager x PORT --model resnet18 --backend fused``
    N worker processes      one ``GpuExperimentWorker`` per GPU (this file, launched by torchrun), each an aiohttp
                            application that registers with the manager, heartbeats, answers ``POST round_start`` /
                            ``POST aggregate`` and reports ``POST update``

A round is triggered exactly like the reference's (``GET /{name}/start_round?n_epoch=K``, manager.py:51-64; the
same call ``baseline/reference_arm.py`` times for the unmodified reference).  HTTP carries metadata only (update
name, ``n_samples``, per-epoch losses, the aggregation plan); the weights stay in the symmetric arena and the
round-end reduce + broadcast is the fused kernel.  The first round also distributes the manager's initial global model
to every seat (it is part of the warm-up).  Every round's shard is copied host->device from pinned memory.

Timing: wall clock on rank 0 around K rounds, bracketed by barrier + synchronize, max over ranks -- the control plane
is host-side by nature.  ``control_plane_ms_per_round`` = round wall time minus the slowest worker's local-training time.
"""
from __future__ import annotations

import asyncio
import os
import subprocess
import sys
import threading
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def main_http(args, emit) -> int:
    import aiohttp
    import torch
    import torch.distributed as dist
    from aiohttp import web

    from .control.gpu_worker import GpuExperimentWorker
    from .data import dirichlet_label_shards, image_shard
    from .models import resnet18

    rank = int(os.environ.get("RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    local_rank = int(os.environ.get("LOCAL_RANK", "0"))
    dev = torch.device("cuda", local_rank)
    torch.cuda.set_device(dev)
    if world > 1 and not dist.is_initialized():
        dist.init_process_group("nccl", device_id=dev)
    # driver-level barriers go through GLOO: an NCCL barrier kernel parked on a worker GPU while rank 0 drives the round
    # would sit beside the fused collective (which needs its whole grid co-resident) and wait for rank 0 -- a cycle
    host_group = dist.new_group(backend="gloo") if world > 1 else None
    name = "resnet18"
    mport = int(os.environ.get("BATON_API_PORT", "18080"))
    wport = mport + 1 + rank

    torch.manual_seed(1000 + rank)          # DIFFERENT init per seat on purpose: the manager's model must win
    model = resnet18(10)
    specs = dirichlet_label_shards(world, 10, args.samples, alpha=args.alpha, seed=11)
    X_host, y_host = image_shard(specs[rank], seed=3, dtype=torch.bfloat16, pin=True)
    h2d = X_host.numel() * X_host.element_size() + y_host.numel() * y_host.element_size()

    def barrier():
        torch.cuda.synchronize()
        if world > 1:
            dist.barrier(group=host_group)
        torch.cuda.synchronize()

    manager_proc = None
    if rank == 0:
        env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
        for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK", "MASTER_ADDR", "MASTER_PORT"):
            env.pop(k, None)
        manager_proc = subprocess.Popen(
            [sys.executable, os.path.join(ROOT, "demo.py"), "manager", "unused", str(mport), "--bind", "127.0.0.1",
             "--model", name, "--backend", args.backend, "--seed", "5"], env=env, stdout=subprocess.DEVNULL)

    loop = asyncio.new_event_loop()
    threading.Thread(target=lambda: (asyncio.set_event_loop(loop), loop.run_forever()), daemon=True).start()

    def call(coro, timeout=600):
        return asyncio.run_coroutine_threadsafe(coro, loop).result(timeout)

    async def manager_get(path):
        async with aiohttp.ClientSession() as s:
            async with s.get("http://127.0.0.1:{}/{}/{}".format(mport, name, path)) as r:
                return r.status, await r.json()

    if rank == 0:
        t0 = time.time()
        while time.time() - t0 < 180:
            try:
                if call(manager_get("clients"))[0] == 200:
                    break
            except Exception:
                time.sleep(0.2)
    barrier()
    state = {}

    async def start_worker():
        app = web.Application(client_max_size=1 << 34)
        w = GpuExperimentWorker(app, model, "127.0.0.1:{}".format(mport), device=dev, shard_fn=lambda: (X_host, y_host),
                                backend=args.backend, wire_dtype=args.wire, port=wport, heartbeat_time=600,
                                worker_host="http://127.0.0.1:{}/{}/".format(wport, name),
                                train_kwargs={"lr": args.lr, "batch_size": args.batch_size},
                                n_ctas=min(args.n_ctas, 132))     # one CTA per SM: slack for foreign kernels
        runner = web.AppRunner(app)
        await runner.setup()
        await web.TCPSite(runner, "127.0.0.1", wport).start()
        state["worker"] = w

    call(start_worker(), timeout=900)        # builds the arena + symmetric-memory session (collective rendezvous)
    t0 = time.time()
    while state["worker"].client_id is None and time.time() - t0 < 120:
        time.sleep(0.05)
    barrier()
    done = {"rounds": 0}

    async def one_round(n_epoch):
        status, accepted = await manager_get("start_round?n_epoch={}".format(n_epoch))
        assert status == 200 and len(accepted) == world and all(accepted.values()), (status, accepted)
        done["rounds"] += 1
        while True:
            _, st = await manager_get("state")
            if not st["in_progress"] and st["n_updates"] >= done["rounds"]:
                _, hist = await manager_get("loss_history")
                return hist[-1] if hist else None
            await asyncio.sleep(0.0005)

    def rounds(k):
        last = None
        for _ in range(k):
            if rank == 0:
                last = call(one_round(args.local_epochs), timeout=900)
            barrier()
        return last

    w = state["worker"]
    try:
        rounds(max(args.warmup, 3))       # round 1 also ships the manager's initial model to every seat
        barrier()
        w.train_seconds = []
        t0 = time.perf_counter()
        last_loss = rounds(args.steps)
        barrier()
        dt = time.perf_counter() - t0
    except BaseException as exc:
        if manager_proc is not None:
            manager_proc.terminate()
        if rank == 0:
            emit({"api": "http", "error": "round failed: {!r}".format(exc)})
        os._exit(1)
    train_s = sum(getattr(w, "train_seconds", []) or [0.0])
    t = torch.tensor([dt, train_s], dtype=torch.float64)
    # every seat must hold the same global model now: checksum the arena
    chk = w.arena.theta[: w.arena.n].double().sum().reshape(1).cpu()
    lo, hi = chk.clone(), chk.clone()
    if world > 1:
        dist.all_reduce(t, op=dist.ReduceOp.MAX, group=host_group)
        dist.all_reduce(lo, op=dist.ReduceOp.MIN, group=host_group)
        dist.all_reduce(hi, op=dist.ReduceOp.MAX, group=host_group)
    dt, train_s = float(t[0]), float(t[1])
    if rank == 0:
        total = world * args.samples * args.local_epochs * args.steps
        emit({
            "api": "http", "impl": "ours",
            "metric": "federated local samples/sec (whole box), ResNet-18 FedAvg, synthetic non-IID 32x32 shards",
            "value": total / dt, "unit": "samples/s", "n_gpus": world, "steps": args.steps,
            "warmup": max(args.warmup, 3), "ms_per_step": dt / args.steps * 1e3, "rounds_per_s": args.steps / dt,
            "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "bf16", "data": "synthetic",
            "timing": "wall clock on rank 0 around GET /start_round ... round closed, barrier+synchronize, max over ranks",
            "config": {"model": "resnet18(num_classes=10)", "global_batch": world * args.batch_size,
                       "batch_size": args.batch_size, "samples_per_client": args.samples,
                       "local_epochs": args.local_epochs, "parallelism": "fedavg dp{}".format(world),
                       "backend": args.backend, "wire_dtype": args.wire,
                       "api": "Manager (CPU process, demo.py manager) + GpuExperimentWorker per GPU over HTTP; "
                              "rounds triggered by GET /start_round"},
            "e2e": {"value": total / dt, "unit": "samples/s", "h2d_bytes_per_step": h2d,
                    "d2h_bytes_per_step": 4 * args.local_epochs},
            "local_train_ms_per_round": train_s / args.steps * 1e3,
            "control_plane_ms_per_round": (dt - train_s) / args.steps * 1e3,
            "replicas_identical": bool(float(lo) == float(hi)),
            "final_loss": last_loss,
        })
    if manager_proc is not None:
        manager_proc.terminate()
    if world > 1:
        dist.destroy_process_group()
    os._exit(0)
