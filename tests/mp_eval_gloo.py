"""CPU / gloo worker for tests/test_eval.py (torchrun --nproc-per-node 2 tests/mp_eval_gloo.py).

``FederatedEngine.evaluate`` across two ranks holding held-out shards of different sizes: the global result must be the
sample-weighted mean of the local results; a rank without a shard contributes nothing; with logical clients every
hosted client's shard is evaluated and summed."""
import math
import os
import sys

import torch
import torch.distributed as dist
from torch import nn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from baton_b200.models import FederatedModule  # noqa: E402
from baton_b200.parallel.engine import FederatedEngine  # noqa: E402


class Tiny(FederatedModule):
    name = "tiny"
    loss_kind = "ce"

    def __init__(self):
        super().__init__()
        self.fc = nn.Linear(6, 4)
        self.bn = nn.BatchNorm1d(4)

    def forward(self, x):
        return self.bn(self.fc(x))


def shard(cid, n):
    g = torch.Generator().manual_seed(500 + cid)
    return torch.randn(n, 6, generator=g), torch.randint(0, 4, (n,), generator=g)


def main():
    dist.init_process_group("gloo")
    rank, world = dist.get_rank(), dist.get_world_size()
    fails = []

    def expect(cond, msg):
        ok = torch.tensor([1 if cond else 0])
        dist.all_reduce(ok, op=dist.ReduceOp.MIN)
        if int(ok) == 0:
            fails.append(msg)
        if rank == 0:
            print(("ok   " if int(ok) else "FAIL ") + msg, flush=True)

    def gathered(res):
        out = [None] * world
        dist.all_gather_object(out, (res.local_loss, res.local_accuracy, res.local_n_samples))
        return out

    def weighted(parts):
        parts = [p for p in parts if p[2] > 0]
        n = sum(p[2] for p in parts)
        return sum(p[0] * p[2] for p in parts) / n, sum(p[1] * p[2] for p in parts) / n, n

    torch.manual_seed(0)
    eng = FederatedEngine(Tiny(), "cpu", backend="nccl", lr=0.1, batch_size=8, name="eval")
    eng.run_round(shard(rank, 32), n_epoch=1)             # the same global model on both ranks afterwards
    sizes = [13, 26]
    res = eng.evaluate(shard(100 + rank, sizes[rank]), batch_size=5)
    loss, acc, n = weighted(gathered(res))
    expect(res.local_n_samples == sizes[rank] and res.n_samples == n == 39, "sample counts (13 + 26)")
    expect(math.isclose(res.loss, loss, rel_tol=1e-9) and math.isclose(res.accuracy, acc, rel_tol=1e-9),
           "global = sample-weighted mean of the local results")

    res = eng.evaluate(shard(100, 13) if rank == 0 else None, batch_size=5)
    parts = gathered(res)
    expect(res.n_samples == 13 and parts[1][2] == 0, "a rank without a shard contributes nothing")
    expect(math.isclose(res.loss, parts[0][0], rel_tol=1e-9), "... and the global result is the other rank's")

    torch.manual_seed(0)
    eng2 = FederatedEngine(Tiny(), "cpu", backend="nccl", lr=0.1, batch_size=8, logical_clients=4, name="logical")
    csizes = {c: 5 + 3 * c for c in range(4)}
    res = eng2.evaluate(lambda c: shard(200 + c, csizes[c]), batch_size=4)
    mine = sum(csizes[c] for c in range(4) if c % world == rank)
    loss, acc, n = weighted(gathered(res))
    expect(res.local_n_samples == mine and res.n_samples == sum(csizes.values()) == n,
           "logical clients: every hosted client's shard is evaluated")
    expect(math.isclose(res.loss, loss, rel_tol=1e-9), "logical clients: global = sample-weighted mean")

    dist.barrier()
    if rank == 0:
        print("RESULT " + ("PASS" if not fails else "FAIL: " + "; ".join(fails)), flush=True)
    dist.destroy_process_group()
    sys.exit(0 if not fails else 1)


if __name__ == "__main__":
    main()
