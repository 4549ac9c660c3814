"""CPU / gloo worker for tests/test_server_opt.py (torchrun --nproc-per-node 2 tests/mp_server_opt_gloo.py).

Two ranks run ``NcclSession`` with FedAdam and FedYogi on gloo for 3 rounds; in round 1 rank 1 hosts no participant
(``n_k = 0``).  After every round each rank's ``global_w``, ``theta``, ``m`` and ``v`` must be bitwise equal to the other
rank's and to the host oracle: ``d = sum_k cast(delta_k * n_k / N)`` (two addends: the order does not matter) and
``apply_update_``."""
import os
import sys

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from baton_b200.models import MLP2  # noqa: E402
from baton_b200.parallel.arena import ParamArena  # noqa: E402
from baton_b200.parallel.fedavg import NcclSession  # noqa: E402
from baton_b200.parallel.server_opt import ServerOptConfig, apply_update_  # noqa: E402


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

    def same_on_every_rank(t):
        ref = t.clone()
        dist.broadcast(ref, 0)
        return torch.equal(t.view(torch.int32), ref.view(torch.int32))

    for kind in ("adam", "yogi"):
        cfg = ServerOptConfig(kind, lr=0.05)
        torch.manual_seed(0)
        arena = ParamArena(MLP2(10, 16, 3), torch.device("cpu"))
        sess = NcclSession(arena, wire_dtype="fp32", mode="delta", server_opt=cfg)
        x = arena.global_w.clone()
        m, v = cfg.init_state(arena.n_param, "cpu")
        for rnd in range(3):
            counts = [3.0, 0.0 if rnd == 1 else 5.0][:world] + [1.0] * (world - 2)
            deltas = [torch.randn(arena.n, generator=torch.Generator().manual_seed(100 * rnd + k)) * 0.01
                      for k in range(world)]
            arena.theta.copy_(arena.global_w + deltas[rank])
            sess.aggregate(my_n=counts[rank])
            total = torch.tensor(counts, dtype=torch.float32).sum()
            d = torch.zeros(arena.n)
            for k in range(world):      # what each rank uploads: cast(src * n_k / N) on the fp32 wire
                d = d + ((x + deltas[k]) - x) * (torch.tensor(counts[k], dtype=torch.float32) / total)
            apply_update_(x, d, arena.n_param, m, v, cfg)
            sm, sv = sess.server_state()
            tag = "{} round {}".format(kind, rnd)
            expect(same_on_every_rank(arena.global_w) and same_on_every_rank(arena.theta) and same_on_every_rank(sm)
                   and same_on_every_rank(sv), tag + ": global_w, theta, m, v identical on every rank")
            expect(torch.equal(arena.global_w.view(torch.int32), x.view(torch.int32)) and torch.equal(sm, m)
                   and torch.equal(sv, v) and torch.equal(arena.theta, x), tag + ": equal to the host oracle")
    dist.barrier()
    if rank == 0:
        print("RESULT", "FAIL" if fails else "PASS", len(fails), flush=True)
    dist.destroy_process_group()
    sys.exit(1 if fails else 0)


if __name__ == "__main__":
    main()
