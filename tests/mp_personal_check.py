"""Multi-GPU worker for tests/test_gpu_personal.py (torchrun --nproc-per-node N tests/mp_personal_check.py, N >= 2).

One client per GPU, ResNet-18 with ``local_keys="bn"`` (FedBN) on the fused collective, fp32 wire, three rounds.  Each
rank snapshots its trained replica when the round's collective is launched and checks that the shared entries agree on
every rank and equal the sample-weighted mean of the snapshots reduced with torch.distributed (the NCCL oracle), and that
the local entries equal this rank's trained values and differ between ranks."""
import os
import sys

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from baton_b200.data import dirichlet_label_shards, image_shard  # noqa: E402
from baton_b200.models import resnet18  # noqa: E402
from baton_b200.parallel.engine import FederatedEngine  # noqa: E402


def main():
    dist.init_process_group("nccl")
    rank, world = dist.get_rank(), dist.get_world_size()
    dev = torch.device("cuda", rank)
    torch.cuda.set_device(dev)
    fails = []

    def expect(cond, msg):
        ok = torch.tensor([1 if cond else 0], device=dev)
        dist.all_reduce(ok, op=dist.ReduceOp.MIN)
        if int(ok) == 0:
            fails.append(msg)
        if rank == 0:
            print(("ok   " if int(ok) else "FAIL ") + msg, flush=True)

    torch.manual_seed(0)
    eng = FederatedEngine(resnet18(10), dev, lr=0.05, batch_size=32, momentum=0.9, wire_dtype="fp32", local_keys="bn")
    a = eng.arena
    lo, hi = a.local_range
    spec = dirichlet_label_shards(world, 10, 64 + 32 * rank, alpha=0.5, seed=1)[rank]
    X, y = image_shard(spec, shift=0.3)
    X, y = X.to(dev, torch.bfloat16), y.to(dev)
    snap = {}
    agg = eng.session.aggregate

    def spy(*args, **kw):
        torch.cuda.current_stream().synchronize()
        snap["t"], snap["g"] = a.theta.clone(), a.global_w.clone()
        return agg(*args, **kw)

    eng.session.aggregate = spy
    for r in range(3):
        eng.run_round((X, y), n_epoch=1)
        eng.sync()
        torch.cuda.synchronize()
        t, g = snap["t"], snap["g"]
        nk = float(X.shape[0])
        num = nk * (torch.cat((t[:lo], t[hi:])) - torch.cat((g[:lo], g[hi:])))
        den = torch.tensor([nk], device=dev)
        dist.all_reduce(num)
        dist.all_reduce(den)
        shared = torch.cat((a.global_w[:lo], a.global_w[hi:]))
        err = float((shared - (torch.cat((g[:lo], g[hi:])) + num / den)).abs().max())
        expect(err < 1e-6, "round {}: shared entries == the NCCL oracle's weighted mean (err {:.1e})".format(r, err))
        other = shared.clone()
        dist.broadcast(other, 0)
        expect(torch.equal(shared, other), "round {}: shared entries agree on every rank".format(r))
        expect(torch.equal(a.theta[lo:hi], t[lo:hi]), "round {}: local entries == this rank's trained values".format(r))
        mine = a.theta[lo:hi].clone()
        first = mine.clone()
        dist.broadcast(first, 0)
        expect(rank == 0 or not torch.equal(mine, first), "round {}: local entries differ between ranks".format(r))

    dist.barrier()
    if rank == 0:
        print("RESULT", "FAIL" if fails else "PASS", len(fails), flush=True)
    dist.destroy_process_group()
    sys.exit(1 if fails else 0)


if __name__ == "__main__":
    main()
