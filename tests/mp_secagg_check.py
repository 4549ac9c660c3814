"""Multi-rank worker for tests/test_gpu_secagg.py (torchrun --nproc-per-node N tests/mp_secagg_check.py, N >= 2).

The fused secure round against ``NcclSession(secagg=...)`` and the host reference ``reference_round`` on the same data:
every rank's keys come from its own X25519 exchange (two sessions, two sets of keys), yet the masks cancel exactly, so
the global models must be bitwise equal.  Rounds on both wire halves, rounds in which only some ranks host a participant
(``n_k = 0``), a round with a server optimizer, and a last round whose alive mask leaves the last rank out (fused
session and host reference only: ``NcclSession`` has no alive mask)."""
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
from baton_b200.parallel.fedavg import FedAvgSession, NcclSession  # noqa: E402
from baton_b200.parallel.secagg import SecAggConfig  # noqa: E402
from baton_b200.parallel.server_opt import ServerOptConfig  # noqa: E402


def main():
    rank = int(os.environ["RANK"])
    world = int(os.environ["WORLD_SIZE"])
    dev = torch.device("cuda", int(os.environ.get("LOCAL_RANK", rank)))
    torch.cuda.set_device(dev)
    dist.init_process_group("nccl", device_id=dev)
    fails = []

    def expect(cond, msg):
        ok = torch.tensor([1 if cond else 0], device=dev)
        dist.all_reduce(ok, op=dist.ReduceOp.MIN)
        if int(ok) == 0:
            fails.append(msg)
        if rank == 0:
            print(("ok   " if int(ok) else "FAIL ") + msg, flush=True)

    def same_on_every_rank(t):
        ref = t.clone()
        dist.broadcast(ref, 0)
        return torch.equal(t.view(torch.int32), ref.view(torch.int32))

    def gather_np(t):
        out = [torch.zeros_like(t) for _ in range(world)]
        dist.all_gather(out, t)
        return [o.cpu().numpy() for o in out]

    cfg = SecAggConfig(8.0)
    keys = {(i, j): [i, j, 5, 6, 7, 8, 9, 10] for i in range(world) for j in range(i + 1, world)}
    for sopt in (None, ServerOptConfig("avgm", lr=1.0, b1=0.5)):
        arenas = {}
        for name in ("fused", "oracle"):
            torch.manual_seed(0)
            arenas[name] = ParamArena(MLP2(72, 250, 6), dev)
        a_f, a_o = arenas["fused"], arenas["oracle"]
        fused = FedAvgSession(a_f, wire_dtype="fp32", mode="delta", n_ctas=16, secagg=cfg, server_opt=sopt)
        oracle = NcclSession(a_o, wire_dtype="fp32", mode="delta", secagg=cfg, server_opt=sopt)
        expect(not fused.use_nvls, "secure rounds run on peer loads")
        for rnd in range(4):
            counts = [float(2 + k) for k in range(world)]
            if rnd == 2:
                counts[0] = 0.0
            if rnd == 3:
                counts = [0.0] * world
                counts[-1] = 4.0
            gen = torch.Generator(device=dev).manual_seed(1000 * rnd + rank)
            delta = torch.randn(a_f.n, device=dev, generator=gen) * (0.05 + 3.0 * (rnd == 1))
            g0 = a_f.global_w.clone()
            for a in (a_f, a_o):
                a.theta.copy_(a.global_w + delta)
            srcs = gather_np(a_f.theta - g0)
            fused.aggregate(my_n=counts[rank])
            oracle.aggregate(my_n=counts[rank])
            torch.cuda.synchronize()
            fused.check()
            tag = "sopt={} round {}".format(sopt.kind if sopt else None, rnd)
            expect(same_on_every_rank(a_f.global_w) and torch.equal(a_f.theta, a_f.global_w),
                   tag + ": fused global identical on every rank")
            expect(torch.equal(a_f.global_w.view(torch.int32), a_o.global_w.view(torch.int32)),
                   tag + ": fused == NcclSession bit for bit")
            if sopt is None:
                d, sat = sa.reference_round(srcs, counts, cfg.range, keys, [rnd, 0, 0])
                ref = (g0.cpu().numpy() + d).astype(np.float32)
                expect(np.array_equal(a_f.global_w.cpu().numpy().view(np.int32), ref.view(np.int32)),
                       tag + ": fused == host reference bit for bit")
                tot = torch.tensor([fused.last_secagg_saturation()], device=dev)
                dist.all_reduce(tot)
                expect(int(tot) == sat, tag + ": saturation counts add up")
        # the alive mask leaves the last rank out: it neither uploads nor receives
        counts = [float(2 + k) for k in range(world)]
        alive = list(range(world - 1))
        delta = torch.randn(a_f.n, device=dev, generator=torch.Generator(device=dev).manual_seed(77 + rank)) * 0.05
        g0 = a_f.global_w.clone()
        a_f.theta.copy_(g0 + delta)
        srcs = gather_np(a_f.theta - g0)
        fused.aggregate(my_n=counts[rank], alive_ranks=alive)
        torch.cuda.synchronize()
        fused.check()
        if sopt is None:
            d, _ = sa.reference_round(srcs[: world - 1], counts[: world - 1], cfg.range, keys, [0, 0, 0])
            ok = (rank == world - 1 and torch.equal(a_f.global_w, g0)) or (
                rank < world - 1 and np.array_equal(a_f.global_w.cpu().numpy(), (g0.cpu().numpy() + d).astype(np.float32)))
            expect(ok, "alive mask without the last rank: live ranks == host reference, the dead rank untouched")
        fused.symm.barrier()
    dist.barrier()
    if rank == 0:
        print("RESULT", "FAIL" if fails else "PASS", len(fails), flush=True)
    dist.destroy_process_group()
    sys.exit(1 if fails else 0)


if __name__ == "__main__":
    main()
