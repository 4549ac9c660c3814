"""CPU / gloo worker for tests/test_robust.py (torchrun --nproc-per-node 3 tests/mp_robust_gloo.py).

Drives :class:`FederatedEngine` with logical clients and a robust aggregator through the ``torch.distributed`` session
on gloo.  After each of 2 rounds the global model must equal ``robust_combine`` over the participants trained one by
one from the round's global model (every rank replays every participant, so no exchange is needed for the oracle)."""
import os
import sys

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from baton_b200.models import MLP2  # noqa: E402
from baton_b200.parallel.engine import FederatedEngine  # noqa: E402
from baton_b200.parallel.robust import RobustConfig, robust_combine  # noqa: E402
from baton_b200.train import run_local_sgd  # noqa: E402

LR, CLIENTS, K = 0.05, 8, 7


def shard(cid):
    g = torch.Generator().manual_seed(5000 + cid)
    X = torch.randn(16, 10, generator=g)
    y = (X @ torch.arange(1, 11, dtype=torch.float32)).unsqueeze(1) * (1 + cid % 3)
    if cid == 5:
        y = -1e3 * y                                 # a client whose update is far out
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

    for kind in ("median", "trimmed_mean"):
        torch.manual_seed(0)
        model = MLP2(10, 16, 1)
        eng = FederatedEngine(model, "cpu", backend="nccl", loss="mse", lr=LR, batch_size=16, wire_dtype="fp32",
                              logical_clients=CLIENTS, sample_k=K, seed=4, aggregator=kind, trim_ratio=0.2)
        cfg = RobustConfig(kind, 0.2)
        for rnd in range(2):
            g0 = torch.cat([p.detach().clone().flatten() for p in model.parameters()])
            state = eng._rng.getstate()
            parts = eng.draw_participants()
            eng._rng.setstate(state)
            deltas = []
            for cid in parts:
                ref = MLP2(10, 16, 1)
                ref.load_state_dict(model.state_dict())
                X, y = shard(cid)
                run_local_sgd(ref, X, y, n_epoch=1, lr=LR, batch_size=16, loss="mse")
                deltas.append(torch.cat([p.detach().flatten() for p in ref.parameters()]) - g0)
            res = eng.run_round(shard, n_epoch=1)
            want = g0 + robust_combine(torch.stack(deltas), cfg)
            got = torch.cat([p.detach().flatten() for p in model.parameters()])
            err = float((got - want).abs().max())
            expect(res.participants == parts and err < 1e-6,
                   "{} round {}: global model == robust_combine over {} clients (err {:.1e})".format(
                       kind, rnd, len(parts), err))
            expect(torch.equal(eng.arena.theta, eng.arena.global_w), "{} round {}: theta == global".format(kind, rnd))

    dist.barrier()
    if rank == 0:
        print("RESULT", "FAIL" if fails else "PASS", len(fails), flush=True)
    dist.destroy_process_group()
    sys.exit(1 if fails else 0)


if __name__ == "__main__":
    main()
