"""CPU / gloo worker for tests/test_personal.py (torchrun --nproc-per-node 2 tests/mp_personal_gloo.py).

Drives :class:`FederatedEngine` with ``local_keys="head"`` (FedPer on ``MLP2``: ``fc2`` stays with each client) through
the ``torch.distributed`` session on gloo, with 6 logical clients of which 3 are sampled per round, and checks every
round against snapshots of each client's replica taken at the start and at the end of its local training:

* the shared entries are equal on both ranks and equal the host's sample-weighted mean of the trained snapshots;
* each participant's local entries equal its trained snapshot, bit for bit; every other client keeps its own;
* a client starts from the initial local values the first time it trains, and from its own last values after that."""
import os
import sys

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from baton_b200.models import MLP2  # noqa: E402
from baton_b200.parallel.engine import FederatedEngine  # noqa: E402

CLIENTS, SAMPLED, ROUNDS = 6, 3, 3


def shard(cid):
    n = 16 + 8 * cid
    g = torch.Generator().manual_seed(3000 + cid)
    X = torch.randn(n, 10, generator=g)
    w = torch.linspace(-1, 1, 10) * (1 + 0.2 * cid)       # a different task per client
    return X, (X @ w).unsqueeze(1) + 0.01 * torch.randn(n, 1, generator=g)


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

    torch.manual_seed(0)
    model = MLP2(10, 16, 1)
    eng = FederatedEngine(model, "cpu", backend="nccl", loss="mse", lr=0.01, batch_size=8, momentum=0.9,
                          wire_dtype="fp32", logical_clients=CLIENTS, sample_k=SAMPLED, seed=7, name="fedper",
                          local_keys="head")
    a = eng.arena
    lo, hi = a.local_range
    init = a.theta[lo:hi].clone()
    start, trained = {}, {}
    train = eng._train_client

    def spy(cid, X, y, n_epoch, first):
        start[cid] = a.theta.clone()
        out = train(cid, X, y, n_epoch, first)
        trained[cid] = a.theta.clone()
        return out

    eng._train_client = spy
    mine = [c for c in range(CLIENTS) if eng.hosted(c)]
    last = {c: init.clone() for c in mine}
    seen = set()
    for r in range(ROUNDS):
        g0 = a.global_w.clone()
        start.clear()
        trained.clear()
        res = eng.run_round(shard, n_epoch=2)
        parts = res.participants
        starts_ok, local_ok = True, True
        for c in mine:
            if c in parts:
                first = c not in seen
                starts_ok &= torch.equal(start[c][lo:hi], init if first else last[c])
                starts_ok &= torch.equal(start[c][:lo], g0[:lo]) and torch.equal(start[c][hi:], g0[hi:])
                last[c] = trained[c][lo:hi].clone()
                seen.add(c)
            got = torch.cat([t.flatten() for t in eng.local_entries(c).values()])
            want = torch.cat([a._view(torch.cat((torch.zeros(lo), last[c])), a.slots[k]).flatten()
                              for k in eng.personal.keys])
            local_ok &= torch.equal(got, want)
        expect(starts_ok, "round {}: each participant starts from the global shared entries and from its own local "
                          "values (the initial ones the first time)".format(r))
        expect(local_ok, "round {}: every client's local entries == its last trained values".format(r))
        # host mean of the shared entries over every participant's trained snapshot
        num = torch.zeros(a.n)
        den = torch.zeros(1)
        for c in mine:
            if c in parts:
                nk = float(shard(c)[0].shape[0])
                num += nk * (trained[c] - g0)
                den += nk
        dist.all_reduce(num)
        dist.all_reduce(den)
        want = g0 + num / den
        shared = torch.cat((a.global_w[:lo], a.global_w[hi:]))
        err = float((shared - torch.cat((want[:lo], want[hi:]))).abs().max())
        expect(err < 1e-5, "round {}: shared entries == host mean of the trained clients (err {:.1e})".format(r, err))
        other = shared.clone()
        dist.broadcast(other, 0)
        expect(torch.equal(shared, other), "round {}: shared entries equal on every rank".format(r))
        sd = eng.state_dict()
        expect(all(torch.equal(sd[k].flatten(), a._view(torch.cat((torch.zeros(lo), init)), a.slots[k]).flatten())
                   for k in eng.personal.keys), "round {}: state_dict() carries the initial local values".format(r))

    dist.barrier()
    if rank == 0:
        print("RESULT", "FAIL" if fails else "PASS", len(fails), flush=True)
    dist.destroy_process_group()
    sys.exit(1 if fails else 0)


if __name__ == "__main__":
    main()
