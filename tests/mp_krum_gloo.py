"""CPU / gloo worker for tests/test_krum.py (torchrun --nproc-per-node 3 tests/mp_krum_gloo.py).

Drives :class:`FederatedEngine` with logical clients and ``aggregator="krum"`` through the ``torch.distributed`` session
on gloo.  Two of the eight clients upload a scaled, sign-flipped update.  After each of 2 rounds the global model must
equal the Krum oracle over the participants trained one by one from the round's global model (every rank replays every
participant), the attackers must be rejected, and every rank must report the same ``last_krum()``."""
import os
import sys

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from baton_b200.models import MLP2  # noqa: E402
from baton_b200.parallel.engine import FederatedEngine  # noqa: E402
from baton_b200.parallel.robust import RobustConfig, krum_select, robust_combine  # noqa: E402
from baton_b200.train import run_local_sgd  # noqa: E402

LR, CLIENTS, K, F = 0.05, 8, 7, 2
ATTACKERS = (2, 5)


def shard(cid):
    g = torch.Generator().manual_seed(7000 + cid)
    X = torch.randn(16, 10, generator=g)
    y = (X @ torch.arange(1, 11, dtype=torch.float32)).unsqueeze(1)
    if cid in ATTACKERS:
        y = -20.0 * y
    return X, y


def main():
    dist.init_process_group("gloo")
    rank = dist.get_rank()
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
    eng = FederatedEngine(model, "cpu", backend="nccl", loss="mse", lr=LR, batch_size=16, wire_dtype="fp32",
                          logical_clients=CLIENTS, sample_k=K, seed=4, aggregator="krum", krum_f=F)
    cfg = RobustConfig("krum", krum_f=F)
    for rnd in range(2):
        g0 = torch.cat([p.detach().clone().flatten() for p in model.parameters()])
        state = eng._rng.getstate()
        parts = eng.draw_participants()
        eng._rng.setstate(state)
        # segment order: ranks in order, then each rank's hosted participants in draw order
        order = [c for r in range(dist.get_world_size()) for c in parts if c % dist.get_world_size() == r]
        deltas = []
        for cid in order:
            ref = MLP2(10, 16, 1)
            ref.load_state_dict(model.state_dict())
            X, y = shard(cid)
            run_local_sgd(ref, X, y, n_epoch=1, lr=LR, batch_size=16, loss="mse")
            deltas.append(torch.cat([p.detach().flatten() for p in ref.parameters()]) - g0)
        stack = torch.stack(deltas)
        res = eng.run_round(shard, n_epoch=1)
        want = g0 + robust_combine(stack, cfg)
        got = torch.cat([p.detach().flatten() for p in model.parameters()])
        err = float((got - want).abs().max())
        expect(res.participants == parts and err < 1e-6,
               "round {}: global model == krum oracle over {} clients (err {:.1e})".format(rnd, len(parts), err))
        kept = krum_select(stack, cfg)[2]
        rep = eng.last_krum()
        expect(sorted(rep) == sorted(parts) and all(rep[c][1] == bool(kept[i]) for i, c in enumerate(order)),
               "round {}: last_krum matches the oracle's kept set".format(rnd))
        expect(not any(rep[c][1] for c in ATTACKERS if c in rep), "round {}: attackers rejected".format(rnd))
        flat = torch.tensor([rep[c][0] for c in sorted(rep)] + [float(rep[c][1]) for c in sorted(rep)],
                            dtype=torch.float64)
        ref0 = flat.clone()
        dist.broadcast(ref0, 0)
        expect(torch.equal(flat, ref0), "round {}: every rank reports the same last_krum".format(rnd))
        expect(torch.equal(eng.arena.theta, eng.arena.global_w), "round {}: theta == global".format(rnd))

    dist.barrier()
    if rank == 0:
        print("RESULT", "FAIL" if fails else "PASS", len(fails), flush=True)
    dist.destroy_process_group()
    sys.exit(1 if fails else 0)


if __name__ == "__main__":
    main()
