"""Multi-rank worker for tests/test_gpu_krum.py (torchrun --nproc-per-node N tests/mp_krum_check.py, N >= 2).

The fused Krum collective against the ``NcclSession`` oracle on the same data, three client segments per rank, over
rounds on both wire halves and one round with the last rank outside the alive mask: the same kept set on every rank and
in the oracle, and a global model bitwise identical across the live ranks and to the oracle's."""
import os
import sys

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from baton_b200.models import MLP2  # noqa: E402
from baton_b200.parallel.arena import ParamArena  # noqa: E402
from baton_b200.parallel.fedavg import FedAvgSession, NcclSession  # noqa: E402
from baton_b200.parallel.robust import RobustConfig  # noqa: E402

S = 3


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
        return torch.equal(t, ref)

    cfg = RobustConfig("krum", krum_f=1)
    for wire in ("fp32", "bf16"):
        arenas = {}
        for name in ("fused", "oracle"):
            torch.manual_seed(0)
            arenas[name] = ParamArena(MLP2(72, 250, 6), dev)
        a_f, a_o = arenas["fused"], arenas["oracle"]
        fused = FedAvgSession(a_f, wire_dtype=wire, mode="delta", n_ctas=16, robust=cfg, max_clients=S)
        oracle = NcclSession(a_o, wire_dtype=wire, mode="delta", robust=cfg, max_clients=S)
        for rnd in range(3):
            alive = list(range(world)) if rnd < 2 else list(range(world - 1))
            live = rank in alive
            gen = torch.Generator(device=dev).manual_seed(1000 * rnd)
            common = torch.randn(a_f.n, device=dev, generator=gen) * 0.01
            for a, sess in ((a_f, fused), (a_o, oracle)):
                g0 = a.global_w.clone()
                for j in range(S):
                    c = rank * S + j                      # well-separated: the noise grows with the client index
                    g = torch.Generator(device=dev).manual_seed(1000 * rnd + c + 1)
                    a.theta.copy_(g0 + common + torch.randn(a.n, device=dev, generator=g) * 0.004 * (1 + 0.45 * c))
                    sess.pack_client(j, reset=j + 1 < S)
            m = S if live else 0
            fused.aggregate(my_n=float(m), n_clients=m, alive_ranks=alive)
            oracle.aggregate(my_n=float(m), n_clients=m)
            torch.cuda.synchronize(dev)
            fused.check()
            tag = "{} round {} ({} live ranks)".format(wire, rnd, len(alive))
            if live:
                kf = fused.last_krum()[2]
                ko = oracle.last_krum()[2]
                kept_ok = kf.tolist() == ko.tolist() and len(kf) == S * len(alive)
                bits_ok = torch.equal(a_f.global_w.view(torch.int32), a_o.global_w.view(torch.int32))
            else:
                kf, kept_ok, bits_ok = None, True, True
            expect(kept_ok, tag + ": fused kept set == NcclSession oracle's")
            expect(bits_ok, tag + ": fused global_w bitwise == oracle")
            probe = a_f.global_w[:4096].clone() if live else torch.zeros(4096, device=dev)
            gathered = [torch.zeros_like(probe) for _ in range(world)]
            dist.all_gather(gathered, probe)
            expect(all(torch.equal(gathered[r].view(torch.int32), gathered[alive[0]].view(torch.int32)) for r in alive),
                   tag + ": global_w identical on every live rank")
            # every rank continues from the live ranks' global model (the oracle also updated the dead rank)
            for a in (a_f, a_o):
                dist.broadcast(a.global_w, alive[0])
                a.theta.copy_(a.global_w)
                a.sync_shadow()
        del fused, oracle
    dist.barrier()
    if rank == 0:
        print("RESULT", "FAIL" if fails else "PASS", len(fails), flush=True)
    dist.destroy_process_group()
    sys.exit(1 if fails else 0)


if __name__ == "__main__":
    main()
