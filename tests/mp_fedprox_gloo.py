"""CPU / gloo worker for tests/test_fedprox.py (torchrun --nproc-per-node 2 tests/mp_fedprox_gloo.py).

Drives :class:`FederatedEngine` with ``prox_mu > 0`` through the ``torch.distributed`` session on gloo and checks the
global model after one round against a hand-computed FedProx local training on every rank followed by the
sample-weighted FedAvg of the results."""
import os
import sys

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from baton_b200.models import MLP2  # noqa: E402
from baton_b200.parallel.engine import FederatedEngine  # noqa: E402

LR, MU, EPOCHS = 0.05, 0.5, 3


def shard(cid, n):
    g = torch.Generator().manual_seed(2000 + cid)
    X = torch.randn(n, 10, generator=g)
    w = torch.arange(1, 11, dtype=torch.float32)
    return X, (X @ w).unsqueeze(1) + 0.01 * torch.randn(n, 1, generator=g)


def fedprox_by_hand(model, X, y, mu):
    """Full-batch local training (one batch per epoch, so the sample order does not matter): w -= lr * (g + mu (w - a))."""
    params = [p.detach().clone().requires_grad_(True) for p in model.parameters()]
    anchor = [p.detach().clone() for p in params]
    for _ in range(EPOCHS):
        h = torch.relu(X @ params[0].t() + params[1])
        loss = torch.nn.functional.mse_loss(h @ params[2].t() + params[3], y)
        grads = torch.autograd.grad(loss, params)
        with torch.no_grad():
            for p, g, a in zip(params, grads, anchor):
                p.sub_(LR * (g + mu * (p - a)))
    return [p.detach() for p in params]


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

    sizes = [24 * (r + 1) for r in range(world)]
    X, y = shard(rank, sizes[rank])
    results = {}
    for mu in (0.0, MU):
        torch.manual_seed(0)
        model = MLP2(10, 16, 1)
        eng = FederatedEngine(model, "cpu", backend="nccl", loss="mse", lr=LR, batch_size=sizes[-1],
                              wire_dtype="fp32", name="prox", prox_mu=mu)
        local = fedprox_by_hand(model, X, y, mu)             # from the global model the round starts from
        eng.run_round((X, y), n_epoch=EPOCHS)
        want = []
        for t in local:
            t = t * (sizes[rank] / sum(sizes))
            dist.all_reduce(t)
            want.append(t)
        got = [p.detach() for p in model.parameters()]
        err = max(float((g - w).abs().max()) for g, w in zip(got, want))
        expect(err < 2e-5, "mu={}: global model == FedAvg of the hand-computed FedProx clients (err {:.1e})".format(
            mu, err))
        expect(torch.equal(eng.arena.theta, eng.arena.global_w), "mu={}: theta == global copy after the round".format(mu))
        results[mu] = torch.cat([w.flatten() for w in want])
    expect(float((results[MU] - results[0.0]).abs().max()) > 1e-3, "the proximal term changes the round's result")

    dist.barrier()
    if rank == 0:
        print("RESULT", "FAIL" if fails else "PASS", len(fails), flush=True)
    dist.destroy_process_group()
    sys.exit(1 if fails else 0)


if __name__ == "__main__":
    main()
