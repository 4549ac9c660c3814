"""Multi-GPU check of the top-k collective (torchrun --nproc-per-node N tests/mp_topk_check.py, N >= 2 GPUs).

Every rank runs a FedAvgSession and an NcclSession (the torch.distributed estimator: dense cast(w * topk(u))
all-reduced) on identical arenas for 3 rounds of top-k 5 % uploads with error feedback, fp32 and bf16 wires; in round 1
rank 1 hosts no participant (n_k = 0).  The global models must agree within the wire's rounding of a reordered sum, the
residuals bit for bit, and every rank must hold the same global model."""
import os
import sys

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from baton_b200.models import MLP2  # noqa: E402
from baton_b200.parallel.arena import ParamArena  # noqa: E402
from baton_b200.parallel.compress import TopKConfig  # noqa: E402
from baton_b200.parallel.fedavg import FedAvgSession, NcclSession  # noqa: E402


def main():
    rank = int(os.environ["RANK"])
    world = int(os.environ["WORLD_SIZE"])
    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    dist.init_process_group("nccl", device_id=dev)
    fails = []

    def expect(cond, msg):
        ok = torch.tensor([1 if cond else 0], device=dev)
        dist.all_reduce(ok, op=dist.ReduceOp.MIN)
        if int(ok) == 0:
            fails.append(msg)
        if rank == 0:
            print(("ok   " if int(ok) else "FAIL ") + msg, flush=True)

    for wire in ("fp32", "bf16"):
        arenas, sessions, res = [], [], []
        for Session in (FedAvgSession, NcclSession):
            torch.manual_seed(0)
            a = ParamArena(MLP2(300, 512, 10), dev)
            kw = {"nvls": False} if Session is FedAvgSession else {}
            sessions.append(Session(a, wire_dtype=wire, mode="delta", topk=TopKConfig(0.05), **kw))
            arenas.append(a)
            res.append(torch.zeros(a.n, device=dev))
        for rnd in range(3):
            n_k = 0.0 if (rnd == 1 and rank == 1) else float(3 + rank)
            gen = torch.Generator(device=dev).manual_seed(100 * rnd + rank)
            d = torch.randn(arenas[0].n, device=dev, generator=gen) * 0.01
            for a, s, e in zip(arenas, sessions, res):
                a.theta.copy_(a.global_w + d)
                if n_k:
                    s.pack_topk(e)
                s.aggregate(my_n=n_k)
            torch.cuda.synchronize()
            sessions[0].check()
            tag = "{} round {}".format(wire, rnd)
            g_f, g_n = arenas[0].global_w, arenas[1].global_w
            tol = 1e-6 if wire == "fp32" else 1e-2
            err = float((g_f - g_n).abs().max() / g_n.abs().max())
            expect(err <= tol, tag + ": fused vs nccl within {} (got {:.2e})".format(tol, err))
            expect(torch.equal(res[0], res[1]), tag + ": residuals bitwise equal")
            ref = g_f.clone()
            dist.broadcast(ref, 0)
            expect(torch.equal(ref, g_f), tag + ": the same global model on every rank")
    dist.barrier()
    if rank == 0:
        print("RESULT", "FAIL" if fails else "PASS", len(fails), flush=True)
    dist.destroy_process_group()
    sys.exit(1 if fails else 0)


if __name__ == "__main__":
    main()
