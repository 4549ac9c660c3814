"""CPU / gloo worker for tests/test_secagg.py (torchrun --nproc-per-node 2..4 tests/mp_secagg_gloo.py).

Every rank runs ``NcclSession(secagg=...)`` on gloo for 3 rounds: the pair keys come from the session's own X25519
exchange, round 1 leaves the last rank without a participant (``n_k = 0``) and round 2 runs FedAvgM.  After every round
each rank's ``global_w`` must be bitwise equal to the other ranks' and to the host reference ``reference_round`` over
every rank's update (whatever the keys: the masks cancel), and within ``P 2^-(f+1)`` plus fp32 rounding of the plain
fp32 mean."""
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from baton_b200.models import MLP2  # noqa: E402
from baton_b200.parallel import secagg as sa  # noqa: E402
from baton_b200.parallel.arena import ParamArena  # noqa: E402
from baton_b200.parallel.fedavg import NcclSession  # noqa: E402
from baton_b200.parallel.secagg import SecAggConfig  # noqa: E402


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

    cfg = SecAggConfig(4.0)
    torch.manual_seed(0)
    arena = ParamArena(MLP2(10, 16, 3), torch.device("cpu"))
    sess = NcclSession(arena, wire_dtype="fp32", mode="delta", secagg=cfg)
    expect(len(sess._secagg_keys) == world - 1, "one pair key per peer")
    for rnd in range(3):
        counts = [float(3 + k) for k in range(world)]
        if rnd == 1:
            counts[-1] = 0.0
        deltas = [(torch.randn(arena.n, generator=torch.Generator().manual_seed(100 * rnd + k)) * 0.3).numpy()
                  for k in range(world)]
        x0 = arena.global_w.clone()
        arena.theta.copy_(x0 + torch.from_numpy(deltas[rank]))
        sess.aggregate(my_n=counts[rank])
        srcs = [((x0 + torch.from_numpy(dk)) - x0).numpy() for dk in deltas]
        d, _ = sa.reference_round(srcs, counts, cfg.range, {(i, j): [i, j, 1, 2, 3, 4, 5, 6] for i in range(world)
                                                             for j in range(i + 1, world)}, [9, 0, 0])
        ref = (x0.numpy() + d).astype(np.float32)
        tag = "round {}".format(rnd)
        expect(same_on_every_rank(arena.global_w) and torch.equal(arena.theta, arena.global_w),
               tag + ": global_w, theta identical on every rank")
        expect(np.array_equal(arena.global_w.numpy().view(np.int32), ref.view(np.int32)),
               tag + ": bit-equal to the host reference with other keys and nonce")
        w, _ = sa.weights(counts)
        terms = [float(w[k]) * np.clip(srcs[k], -cfg.range, cfg.range).astype(np.float64) for k in range(world)]
        mean = sum(terms)
        P = sum(1 for c in counts if c > 0)
        # each participant rounds to 2^-f once; w_k y_k and the decode round in fp32
        tol = P * 2.0 ** -(cfg.frac_bits + 1) + 2.0 ** -22 * (sum(np.abs(t) for t in terms) + np.abs(mean))
        expect(bool(np.all(np.abs(d - mean) <= tol)), tag + ": within P 2^-(f+1) of the fp32 mean")
    dist.barrier()
    if rank == 0:
        print("RESULT", "FAIL" if fails else "PASS", len(fails), flush=True)
    dist.destroy_process_group()
    sys.exit(1 if fails else 0)


if __name__ == "__main__":
    main()
