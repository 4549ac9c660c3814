"""Multi-rank worker for the distributed tier (launched by torchrun from test_gpu_fedavg.py or by
hand:  torchrun --nproc-per-node 2 --master-addr 127.0.0.1 tests/mp_fedavg_check.py).

Checks the fused NVLink FedAvg kernel against the closed-form FedAvg formula and the NCCL oracle:
bf16/fp32/block-scaled-fp8 wire, delta/weights upload, counts on the barrier flags vs host plan, partial
participation (n_k = 0), a rank excluded by the alive mask, NVLS on/off, integer side arena (max),
loss-history reduce, momentum reset, and the flag-gated first GEMM (bcast_gemm)."""
import os
import sys

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from baton_b200.ops import functional as F  # noqa: E402
from baton_b200.ops import nn as bnn  # noqa: E402
from baton_b200.parallel.arena import ParamArena  # noqa: E402
from baton_b200.parallel.fedavg import FedAvgSession, NcclSession  # noqa: E402

BF16 = torch.bfloat16


class Net(torch.nn.Module):
    def __init__(self):
        super().__init__()
        self.fc1 = bnn.Linear(512, 1024, act="relu")
        self.bn = bnn.BatchNorm2d(64)
        self.fc2 = bnn.Linear(1024, 16, out_fp32=True)

    def forward(self, x):
        return self.fc2(self.fc1(x))


def log(rank, *a):
    if rank == 0:
        print(*a, flush=True)


def main():
    rank = int(os.environ["RANK"])
    world = int(os.environ["WORLD_SIZE"])
    dev = torch.device("cuda", int(os.environ.get("LOCAL_RANK", rank)))
    torch.cuda.set_device(dev)
    dist.init_process_group("nccl", device_id=dev)
    failures = []

    def expect(cond, msg):
        ok = torch.tensor([1 if cond else 0], device=dev)
        dist.all_reduce(ok, op=dist.ReduceOp.MIN)
        if int(ok) == 0:
            failures.append(msg)
            log(rank, "FAIL", msg)
        else:
            log(rank, "ok  ", msg)

    def gather_all(t):
        out = [torch.empty_like(t) for _ in range(world)]
        dist.all_gather(out, t)
        return out

    for wire in ("fp32", "bf16", "fp8"):
        for mode in ("weights", "delta"):
            for nvls in (False, True):
                if wire == "fp8" and (nvls or mode == "weights"):
                    continue               # block scales need the P2P path; fp8 is meant for deltas
                torch.manual_seed(0)
                net = Net()
                arena = ParamArena(net, dev, momentum=True)
                sess = FedAvgSession(arena, wire_dtype=wire, mode=mode, nvls=nvls, n_ctas=16, tile_flags=True)
                if nvls and not sess.use_nvls:
                    log(rank, "skip NVLS ({}, {}): no multicast support".format(wire, mode))
                    continue
                tag = "{}/{}/{}".format(wire, mode, "nvls" if sess.use_nvls else "p2p")
                g0 = arena.global_w.clone()
                # every rank drifts away from the global model differently
                torch.manual_seed(100 + rank)
                arena.theta.add_(torch.randn_like(arena.theta) * 0.01)
                arena.momentum.fill_(1.0)
                net.bn.num_batches_tracked.fill_(10 + rank)
                n_k = float(100 * (rank + 1))
                thetas = gather_all(arena.theta.clone())
                N = sum(100.0 * (r + 1) for r in range(world))
                want = sum(t * (100.0 * (r + 1) / N) for r, t in enumerate(thetas))
                losses = [float(rank + 1), float(2 * rank + 1)]
                sess.loss_local.zero_()
                sess.loss_local[:2] = torch.tensor(losses, device=dev)
                sess.aggregate(my_n=n_k)                       # counts ride on the barrier flags
                torch.cuda.synchronize()
                sess.check()
                # bf16 wire: one rounding of the value on the wire (|theta| ~ 1 -> 2^-8; |delta| ~ 0.05 -> 2e-4)
                tol = 8e-3 if wire == "bf16" and mode == "weights" else (6e-4 if wire == "bf16" else 1e-6)
                if wire == "fp8":
                    tol = 8e-3             # |delta| <~ 0.05, two e4m3 roundings (2^-4 each) of the block maximum
                err = float((arena.theta - want).abs().max())
                expect(err < tol, "{} weighted mean (err {:.2e})".format(tag, err))
                expect(torch.equal(arena.theta, arena.global_w), tag + " global copy == theta")
                expect(torch.equal(arena.theta_bf16, arena.theta.to(BF16)), tag + " bf16 shadow in sync")
                same = gather_all(arena.theta.clone())
                expect(all(torch.equal(same[0], s) for s in same), tag + " replicas bit-identical")
                expect(float(arena.momentum.abs().max()) == 0.0, tag + " momentum reset")
                expect(int(net.bn.num_batches_tracked) == 10 + world - 1, tag + " int buffer = max")
                wl = [sum((r + 1) * 100.0 * (r + 1) for r in range(world)) / N,
                      sum((2 * r + 1) * 100.0 * (r + 1) for r in range(world)) / N]
                got = sess.reduced_loss(2)
                expect(abs(got[0] - wl[0]) < 1e-4 and abs(got[1] - wl[1]) < 1e-4, tag + " loss history reduce")
                n_flags = -(-arena.n // sess.FLAG_GRANULE)      # one flag per 1024-element granule, whatever the tile size
                expect(int(sess.tile_flags[:n_flags].min()) == 1, tag + " tile flags published")

                # partial participation: the last rank reports n_k = 0 (host plan path)
                torch.manual_seed(200 + rank)
                arena.theta.add_(torch.randn_like(arena.theta) * 0.01)
                thetas = gather_all(arena.theta.clone())
                plan = [100.0 * (r + 1) for r in range(world)]
                plan[-1] = 0.0
                Np = sum(plan)
                want = sum(t * (p / Np) for t, p in zip(thetas, plan))
                sess.aggregate(n_samples_by_rank=plan)
                torch.cuda.synchronize()
                err = float((arena.theta - want).abs().max())
                expect(err < tol, "{} partial participation (err {:.2e})".format(tag, err))

                # a seat excluded by the alive mask is neither read, written nor waited for
                if world > 2 or True:
                    torch.manual_seed(300 + rank)
                    arena.theta.add_(torch.randn_like(arena.theta) * 0.01)
                    before = arena.theta.clone()
                    thetas = gather_all(before)
                    alive = list(range(world - 1)) if world > 1 else [0]
                    plan = [100.0 * (r + 1) if r in alive else 0.0 for r in range(world)]
                    Np = sum(plan)
                    want = sum(t * (p / Np) for t, p in zip(thetas, plan))
                    sess.aggregate(n_samples_by_rank=plan, alive_ranks=alive)
                    torch.cuda.synchronize()
                    if rank in alive:
                        err = float((arena.theta - want).abs().max())
                        good = err < tol
                    else:
                        good = torch.equal(arena.theta, before)
                        # re-join: adopt the global model from rank 0 so later rounds line up again
                    expect(good, tag + " alive-mask subset")
                    dist.broadcast(arena.theta, 0)
                    arena.commit_global()
                    ep = torch.tensor([sess.epoch], device=dev)
                    dist.all_reduce(ep, op=dist.ReduceOp.MAX)
                    sess.epoch = int(ep)
                del sess, arena, net
                torch.cuda.synchronize()
                dist.barrier()

    # NCCL oracle equivalence on the delta/bf16 product configuration
    torch.manual_seed(0)
    net_a = Net()
    torch.manual_seed(0)
    net_b = Net()                      # identical initial weights
    ar_a, ar_b = ParamArena(net_a, dev), ParamArena(net_b, dev)
    fused, oracle = FedAvgSession(ar_a, n_ctas=32), NcclSession(ar_b)
    torch.manual_seed(400 + rank)
    d = torch.randn_like(ar_a.theta) * 0.01
    ar_a.theta.add_(d)
    ar_b.theta.add_(d)
    fused.aggregate(my_n=float(50 + rank))
    oracle.aggregate(my_n=float(50 + rank))
    torch.cuda.synchronize()
    err = float((ar_a.theta - ar_b.theta).abs().max())
    expect(err < 6e-4, "fused == NCCL oracle (err {:.2e})".format(err))

    # bcast_gemm: first GEMM of the next forward gated on per-tile arrival flags, launched while the
    # collective is still running on the high-priority stream
    torch.manual_seed(0)
    net = Net()
    arena = ParamArena(net, dev)
    sess = FedAvgSession(arena, n_ctas=16, tile_flags=True)
    torch.manual_seed(500 + rank)
    arena.theta.add_(torch.randn_like(arena.theta) * 0.01)
    x = torch.randn(256, 512, device=dev).to(BF16)
    sess.aggregate(my_n=1.0, on_side_stream=True)
    sess.gate_first_layer(net.fc1)
    y = net.fc1(x)                     # wgmma GEMM whose TMA producer acquires the tile flags
    sess.join()
    torch.cuda.synchronize()
    ref = torch.relu(x.float() @ net.fc1.weight.detach().to(BF16).float().t() + net.fc1.bias.detach())
    err = float((y.float() - ref).abs().max() / ref.abs().max())
    expect(err < 2e-2, "bcast_gemm consumes the freshly broadcast weights (err {:.2e})".format(err))

    # fault injection: a peer that never joins the collective must turn into an error status on the
    # waiting ranks (bounded spin), not a hang -- and the session must be usable again afterwards
    if os.environ.get("BATON_CHECK_SKIP_DEAD_PEER") == "1":      # under compute-sanitizer the bounded spin takes minutes
        log(rank, "skip dead-peer injection (BATON_CHECK_SKIP_DEAD_PEER=1)")
        dist.barrier()
        if rank == 0:
            print("RESULT", "PASS" if not failures else "FAIL", len(failures), flush=True)
        dist.destroy_process_group()
        sys.exit(1 if failures else 0)
    torch.manual_seed(0)
    net = Net()
    arena = ParamArena(net, dev)
    sess = FedAvgSession(arena, n_ctas=8, timeout_log2=20)
    timed_out = True
    if rank != world - 1:                      # the last rank "dies": it skips this round
        sess.aggregate(my_n=1.0)
        torch.cuda.synchronize()
        try:
            sess.check()
            timed_out = False
        except RuntimeError:
            timed_out = True
    expect(timed_out, "dead peer -> timeout status instead of a hang")
    ep = torch.tensor([sess.epoch], device=dev)
    dist.all_reduce(ep, op=dist.ReduceOp.MAX)
    sess.epoch = int(ep)
    dist.broadcast(arena.theta, 0)
    arena.commit_global()
    torch.manual_seed(600 + rank)
    arena.theta.add_(torch.randn_like(arena.theta) * 0.01)
    thetas = gather_all(arena.theta.clone())
    sess.aggregate(my_n=1.0)
    torch.cuda.synchronize()
    sess.check()
    err = float((arena.theta - sum(thetas) / world).abs().max())
    expect(err < 6e-4, "session recovers after the timeout (err {:.2e})".format(err))

    dist.barrier()
    if rank == 0:
        print("RESULT", "FAIL" if failures else "PASS", len(failures), flush=True)
    dist.destroy_process_group()
    sys.exit(1 if failures else 0)


if __name__ == "__main__":
    main()
