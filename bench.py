#!/usr/bin/env python
"""Flagship benchmark: ResNet-18 FedAvg on H100, one federated client per GPU.

    python bench.py --gpus N --steps K --warmup W           (N > 1: launched under torchrun)
    python bench.py ... --dump-outputs DIR                   (also write what the last timed round computed)

One *step* is one federated round:
    local SGD over the client's private synthetic non-IID shard (local_epochs=1, bf16)
    -> fused weighted reduce + broadcast + running-mean apply over NVLink (ONE kernel, no NCCL)
``value`` = local samples/s summed over all N clients (weak scaling: per-client work is fixed),
device-timed with CUDA events, max over ranks.  ``e2e`` repeats the measurement through the public
API (``FederatedEngine.run_round``) with the shard copied host->device from pinned memory and the
per-epoch loss read back device->host EVERY round.

``--impl reference`` runs the unmodified reference (baseline/reference_arm.py, nothing of this
package on that path); ``--impl baseline`` runs the same algorithm on stock PyTorch ops with the
round-end reduce done by NCCL.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
DUMP_MAX_ELEMS = 16 << 20          # 64 MB of float32


def parse_args(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--impl", default="ours", choices=["ours", "reference", "baseline"])
    ap.add_argument("--model", default="resnet18", choices=["resnet18", "resnet50", "bert_base", "bert_tiny"])
    ap.add_argument("--seq-len", type=int, default=128)
    ap.add_argument("--batch-size", type=int, default=128)
    ap.add_argument("--samples", type=int, default=4096, help="samples per client per round")
    ap.add_argument("--local-epochs", type=int, default=1)
    ap.add_argument("--lr", type=float, default=0.05)
    ap.add_argument("--momentum", type=float, default=0.0)
    ap.add_argument("--alpha", type=float, default=0.5, help="Dirichlet label skew of the shards")
    ap.add_argument("--wire", default="bf16", choices=["bf16", "fp32", "fp8"],
                    help="wire format of the fused FedAvg collective (fp8 = e4m3 + UE8M0 scale per 32 elements)")
    ap.add_argument("--dtype", default="bf16", choices=["bf16", "fp8"],
                    help="fp8 = block-scaled MXFP8 convolutions (fwd/dgrad/wgrad), everything else bf16/fp32")
    ap.add_argument("--backend", default="fused", choices=["fused", "nccl"])
    ap.add_argument("--n-ctas", type=int, default=132)
    ap.add_argument("--no-graph", action="store_true")
    ap.add_argument("--bcast-gemm", type=int, default=int(os.environ.get("BATON_BCAST_GEMM", "0")),
                    help="1: K3 -- the head of the next round's captured epoch (batch gather, im2col, flag-gated weight staging "
                         "+ first conv GEMM) runs while the round-end collective is still in flight")
    ap.add_argument("--api", default="engine", choices=["engine", "http"],
                    help="http: drive the rounds through Manager + GpuExperimentWorker over HTTP (GET /start_round), "
                         "one worker process per GPU and a CPU manager process -- Baton's API on the NVLink data plane")
    ap.add_argument("--graph", action="store_true",
                    help="--impl baseline only: CUDA-graph the stock model's local epoch + flat-buffer NCCL aggregate")
    ap.add_argument("--nvls", default="auto")
    ap.add_argument("--logical-clients", type=int, default=0,
                    help="> n_gpus: time-slice this many logical clients over the GPUs (sampling sweep config)")
    ap.add_argument("--sample-k", type=int, default=None, help="logical clients sampled per round")
    ap.add_argument("--dump-outputs", metavar="DIR", default=None,
                    help="after the timed rounds, write the global model the last one produced to DIR/*.npy (float32; "
                         "a fixed seeded sample above %d parameters) so two builds can be compared output for output"
                         % DUMP_MAX_ELEMS)
    return ap.parse_args(argv)


class ClockSampler:
    """nvidia-smi sampler running DURING the timed region (SM clock, power, throttle reasons)."""

    Q = ("index,clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.hw_slowdown,"
         "clocks_event_reasons.hw_thermal_slowdown,clocks_event_reasons.sw_thermal_slowdown,"
         "clocks_event_reasons.sw_power_cap")

    def __init__(self, gpu_index: int):
        self.gpu_index = gpu_index
        self.proc = None
        self.path = "/tmp/bench_clocks_{}.csv".format(os.getpid())

    def start(self):
        try:
            self.proc = subprocess.Popen(
                ["nvidia-smi", "--query-gpu=" + self.Q, "--format=csv,noheader,nounits", "-lms", "100",
                 "-i", str(self.gpu_index)], stdout=open(self.path, "w"), stderr=subprocess.DEVNULL)
        except Exception:
            self.proc = None

    def stop(self) -> dict:
        if self.proc is None:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["nvidia-smi unavailable"]}
        self.proc.terminate()
        try:
            self.proc.wait(timeout=5)
        except Exception:
            self.proc.kill()
        sm, mx, reasons, power = [], [], set(), []
        try:
            for line in open(self.path):
                f = [x.strip() for x in line.split(",")]
                if len(f) < 8:
                    continue
                try:
                    sm.append(float(f[1])); mx.append(float(f[2])); power.append(float(f[3]))
                except ValueError:
                    continue
                for name, v in zip(("hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"), f[4:8]):
                    if v.lower().startswith("active"):
                        reasons.add(name)
        except OSError:
            pass
        return {"sm_mhz": statistics.median(sm) if sm else None, "sm_max_mhz": max(mx) if mx else None,
                "power_w_max": max(power) if power else None, "samples": len(sm), "reasons": sorted(reasons)}


def _claim_stdout():
    """Everything written to fd 1 from here on (NCCL's version banner, library chatter) goes to stderr;
    the returned fd is the real stdout, used once for the single JSON result line."""
    sys.stdout.flush()
    real = os.dup(1)
    os.dup2(2, 1)
    return real


def _emit(real_fd: int, obj) -> None:
    os.write(real_fd, (json.dumps(obj) + "\n").encode())


def _dump_outputs(out_dir: str, arena) -> None:
    """The global model after the last timed round -- what ``run_round`` hands the next round and the caller --
    as float32 .npy.  Models above DUMP_MAX_ELEMS parameters are sampled at fixed positions: an even stride with a
    seeded offset inside each stride, so the sample costs O(DUMP_MAX_ELEMS) and is the same in every run."""
    import numpy as np
    import torch
    w = (arena.global_w if arena.global_w is not None else arena.theta)[: arena.n_param].detach().float()
    n = w.numel()
    if n > DUMP_MAX_ELEMS:
        stride = n // DUMP_MAX_ELEMS
        g = torch.Generator().manual_seed(0)
        idx = torch.arange(DUMP_MAX_ELEMS, dtype=torch.int64) * stride + torch.randint(0, stride, (DUMP_MAX_ELEMS,), generator=g)
        w = w[idx.to(w.device)]
    os.makedirs(out_dir, exist_ok=True)
    np.save(os.path.join(out_dir, "global_weights.npy"), w.cpu().numpy().astype(np.float32))


def main(argv=None):
    args = parse_args(argv)
    if args.impl == "reference":
        os.execv(sys.executable, [sys.executable, os.path.join(ROOT, "baseline", "reference_arm.py")] + sys.argv[1:])
    if args.impl == "baseline":
        os.execv(sys.executable, [sys.executable, os.path.join(ROOT, "baseline", "nccl_fedavg.py")] + sys.argv[1:])

    real_stdout = _claim_stdout()
    if args.api == "http":
        sys.path.insert(0, ROOT)
        from baton_b200.apibench import main_http
        return main_http(args, lambda obj: _emit(real_stdout, obj))
    import torch
    import torch.distributed as dist

    rank = int(os.environ.get("RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    local_rank = int(os.environ.get("LOCAL_RANK", "0"))
    if not torch.cuda.is_available():
        if rank == 0:
            _emit(real_stdout, {"metric": "federated local samples/sec", "value": None, "error": "no CUDA device"})
        return 1
    dev = torch.device("cuda", local_rank)
    torch.cuda.set_device(dev)
    if world > 1:
        dist.init_process_group("nccl", device_id=dev)

    sys.path.insert(0, ROOT)
    from baton_b200.data import dirichlet_label_shards, image_shard, token_shard
    from baton_b200.models import bert_base, bert_tiny, resnet18, resnet50
    from baton_b200.ops._ext import launch_counts, total_launches
    from baton_b200.parallel.engine import FederatedEngine

    torch.manual_seed(0)   # same init on every rank == the global model every client starts from
    if args.model == "resnet18":
        model = resnet18(10)
    elif args.model == "resnet50":
        model = resnet50(1000 if args.samples >= 1000 else 10)
    elif args.model == "bert_base":
        model = bert_base(2)
    else:
        model = bert_tiny(2)
    is_bert = args.model.startswith("bert")
    if args.dtype == "fp8":
        model.set_precision("fp8")
    eng = FederatedEngine(model, dev, backend=args.backend, lr=args.lr, batch_size=args.batch_size,
                          momentum=args.momentum, wire_dtype=args.wire, n_ctas=args.n_ctas,
                          use_graph=not args.no_graph, nvls=(args.nvls if args.nvls == "auto" else args.nvls == "1"),
                          name=args.model, logical_clients=args.logical_clients, sample_k=args.sample_k, seed=5,
                          tile_flags=bool(args.bcast_gemm))

    # private synthetic non-IID shard of this client, in pinned host memory (bf16 NHWC) + resident copy
    num_classes = model.config.num_labels if is_bert else model.fc.out_features
    n_logical = args.logical_clients if args.logical_clients > world else world
    specs = dirichlet_label_shards(n_logical, num_classes, args.samples, alpha=args.alpha, seed=11)
    mine = [c for c in range(n_logical) if c % world == rank]
    if is_bert:
        host_shards = {c: token_shard(specs[c], seq_len=args.seq_len, vocab=model.config.vocab_size, seed=3, pin=True)
                       for c in mine}
    else:
        host_shards = {c: image_shard(specs[c], seed=3, dtype=torch.bfloat16, pin=True) for c in mine}
    dev_shards = {c: (x.to(dev), y.to(dev)) for c, (x, y) in host_shards.items()}
    X_host, y_host = host_shards[mine[0]]
    X_dev, y_dev = dev_shards[mine[0]]
    if eng.logical_clients:      # shards are addressed by logical client id
        X_dev = y_dev = None
        resident = lambda cid: dev_shards[cid]      # noqa: E731
        pinned = lambda cid: host_shards[cid]       # noqa: E731
    h2d = FederatedEngine.h2d_bytes(X_host, y_host)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)   # > 50 MB L2

    def barrier():
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()

    def run(shard, k, read_loss, timers=None):
        last = None
        for i in range(k):
            flush.zero_()                       # evict L2 between rounds (inputs are smaller than L2)
            if timers is not None:
                timers[i][0].record()
            last = eng.run_round(shard, n_epoch=args.local_epochs, read_loss=read_loss)
            if timers is not None:
                timers[i][1].record()
        return last

    # ---- warm-up (captures the epoch graph, warms NVLink mappings) -------------------------------
    res_shard = resident if eng.logical_clients else (X_dev, y_dev)
    pin_shard = pinned if eng.logical_clients else (X_host, y_host)
    if eng.logical_clients:      # capture the epoch graph of every hosted logical client up front
        for c in mine:
            eng.trainer.run(*dev_shards[c], n_epoch=1, return_device=True, **eng.hp)
            eng.arena.theta.copy_(eng.arena.global_w)
            eng.arena.sync_shadow()
    run(res_shard, max(args.warmup, 3), read_loss=False)
    barrier()

    # ---- (a) device-timed: resident shard, no host traffic in the loop ---------------------------
    sampler = ClockSampler(local_rank)
    c_before = total_launches()
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(args.steps)]
    agg_ev = []
    if rank == 0:
        sampler.start()
    barrier()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    n0 = eng.samples_trained
    run(res_shard, args.steps, read_loss=False, timers=ev)
    trained = eng.samples_trained - n0
    eng.sync()          # the last round's collective runs on the side stream: it belongs inside the timed region
    e1.record()
    barrier()
    dev_ms = e0.elapsed_time(e1)
    clocks = sampler.stop() if rank == 0 else None
    if args.dump_outputs and rank == 0:
        _dump_outputs(args.dump_outputs, eng.arena)
    launches = total_launches() - c_before
    kpe = getattr(eng.trainer, "kernels_per_epoch", 0) or 0
    graph_launches = args.steps * args.local_epochs * kpe     # kernels replayed from the captured epoch graph
    gpu_launches = launches + graph_launches

    # ---- exposed aggregate+broadcast time: the fused collective alone, device-timed -------------
    agg_ms = []
    for _ in range(5):
        a0, a1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        barrier()
        eng.sync()
        a0.record()
        eng.session.aggregate(my_n=float(args.samples))
        a1.record()
        torch.cuda.synchronize()
        agg_ms.append(a0.elapsed_time(a1))
    agg_us = min(agg_ms) * 1e3
    link_gbps = None
    symm = getattr(eng.session, "symm", None)
    if world > 1 and symm is not None and hasattr(symm, "measure_link_gbps"):
        try:
            link_gbps = symm.measure_link_gbps()
        except Exception as e:              # evidence only: never fail the bench over it
            sys.stderr.write("link measurement failed: {}\n".format(e))

    # ---- (b) end to end through the public API: pinned H2D every round + loss D2H every round ----
    if eng.logical_clients:      # warm-up: capture the epoch graph over every staging slot a sampled round can use
        eng.sync()
        for j, c in enumerate(mine):
            Xs, ys = eng.stage(*host_shards[c], slot=j)
            eng.trainer.run(Xs, ys, n_epoch=1, return_device=True, **eng.hp)
            eng.arena.theta.copy_(eng.arena.global_w)
            eng.arena.sync_shadow()
    run(pin_shard, 2, read_loss=True)
    barrier()
    n0 = eng.samples_trained
    t0 = time.perf_counter()
    res = run(pin_shard, args.steps, read_loss=True)
    barrier()
    e2e_s = time.perf_counter() - t0
    trained_e2e = eng.samples_trained - n0

    t = torch.tensor([dev_ms, e2e_s * 1e3, agg_us], device=dev, dtype=torch.float64)
    cnt = torch.tensor([trained, trained_e2e], device=dev, dtype=torch.float64)
    if world > 1:
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        dist.all_reduce(cnt, op=dist.ReduceOp.SUM)
    dev_ms, e2e_ms, agg_us = [float(x) for x in t.tolist()]
    if rank == 0:
        value = float(cnt[0]) * args.local_epochs / (dev_ms / 1e3)          # samples actually trained, whole box
        e2e_value = float(cnt[1]) * args.local_epochs / (e2e_ms / 1e3)
        wire_bytes = eng.session.wire_bytes()
        out = {
            "metric": "federated local samples/sec (whole box), {} FedAvg, synthetic non-IID {} shards".format(
                {"resnet18": "ResNet-18", "resnet50": "ResNet-50", "bert_base": "BERT-base", "bert_tiny": "BERT-tiny"}[args.model],
                "seq-{} token".format(args.seq_len) if is_bert else "32x32"),
            "value": value, "unit": "samples/s", "n_gpus": world, "steps": args.steps, "warmup": max(args.warmup, 3),
            "ms_per_step": dev_ms / args.steps, "rounds_per_s": args.steps / (dev_ms / 1e3),
            "higher_is_better": True, "scaling": "weak", "vs_baseline": None,
            "dtype": "bf16" if args.dtype == "bf16" else "mxfp8 convs (e4m3 + ue8m0/32) + bf16", "data": "synthetic",
            "config": {"model": "{}(num_classes={})".format(args.model, num_classes),
                       "global_batch": world * args.batch_size, "batch_size": args.batch_size,
                       "samples_per_client": args.samples, "image": None if is_bert else "32x32x3 NHWC",
                       "seq_len": args.seq_len if is_bert else None,
                       "local_epochs": args.local_epochs, "parallelism": "fedavg dp{}".format(world),
                       "backend": args.backend, "wire_dtype": args.wire, "upload": "delta",
                       "nvls": bool(getattr(eng.session, "use_nvls", False)),
                       "nvls_choice": getattr(eng.session, "nvls_choice", None),
                       "bcast_gemm": bool(getattr(eng, "k3", False)),
                       "upload_copy_emitted_by_sgd": bool(getattr(eng.session, "last_prepacked", False)),
                       "cuda_graph": not args.no_graph, "optimizer": "sgd(lr={}, momentum={})".format(args.lr, args.momentum),
                       "l2": "256 MiB memset between rounds (flush)", "dirichlet_alpha": args.alpha,
                       "logical_clients": n_logical, "sampled_per_round": args.sample_k or n_logical},
            "clocks": clocks,
            "e2e": {"value": e2e_value, "unit": "samples/s", "ms_per_step": e2e_ms / args.steps,
                    "h2d_bytes_per_step": h2d, "d2h_bytes_per_step": 4 * args.local_epochs,
                    "api": "FederatedEngine.run_round(pinned shard) -> RoundResult.loss_history"},
            "gpu_launches": int(gpu_launches),
            "kernels_per_local_step": getattr(eng.trainer, "n_kernels_per_step", None),
            "agg_bcast_us_per_round": agg_us,
            "agg_bcast_wire_bytes": wire_bytes,
            "agg_bcast_roofline": _roofline(agg_us, wire_bytes, world, link_gbps),
            "nvlink_GBps_per_dir_measured_here": link_gbps,
            "final_loss": (res.loss_history[-1] if res and res.loss_history else None),
            "launch_breakdown": dict(launch_counts()),
        }
        _emit(real_stdout, out)
    if world > 1:
        dist.destroy_process_group()
    return 0


def _roofline(agg_us: float, wire_bytes: int, world: int, link_gbps=None):
    """Fraction of the NVLink roofline achieved by the fused reduce+broadcast: bytes that must cross
    one GPU's links in each direction = (K-1)/K * |wire| (reduce-scatter pull and broadcast push use opposite
    directions), over the per-direction bandwidth measured on THIS box by ``SymmetricBuffer.measure_link_gbps``
    (fallback: 450 GB/s, half the 900 GB/s NVLink of the H100 SXM data sheet).  For K = 1 the bound is local HBM
    (3.35 TB/s, H100 SXM data sheet)."""
    if agg_us <= 0:
        return None
    if world <= 1:
        bytes_hbm = wire_bytes * (2 + 2 + 2 + 2 + 1)   # pack r/w, reduce r/w, apply: read wire, write theta/global/bf16
        floor_us = bytes_hbm / 3.35e12 * 1e6
        return {"bound": "hbm", "floor_us": floor_us, "fraction_of_measured": floor_us / agg_us}
    inbound = (world - 1) / world * wire_bytes
    bw = (link_gbps or 450.0) * 1e9
    floor_us = inbound / bw * 1e6             # pull and push use opposite directions concurrently
    return {"bound": "nvlink {:.0f} GB/s/dir ({})".format(bw / 1e9, "measured in this run" if link_gbps else "H100 SXM data sheet"),
            "floor_us": floor_us, "fraction_of_measured": floor_us / agg_us}


if __name__ == "__main__":
    sys.exit(main())
