"""Multi-rank worker for tests/test_gpu_server_opt.py (torchrun --nproc-per-node N tests/mp_server_opt_check.py, N >= 2).

FedAdam and FedYogi on the fused collective against the ``NcclSession`` oracle on the same data, over rounds on both
wire halves, on peer loads and with ``nvls=True`` (the multicast reduce wherever the box has NVLS multicast;
there the step reads ``apply_scale = 1 / (N * prescale)``), and rounds in which only some ranks host a participant
(``sample_k < world``): the global model and the
server state bitwise identical on every rank, and equal to the oracle's to the rounding of the reduction (the fused
collective weighs on the reader side in rank order, NCCL sums pre-weighted wire values in its own order)."""
import os
import sys

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from baton_b200.models import MLP2  # noqa: E402
from baton_b200.parallel.arena import ParamArena  # noqa: E402
from baton_b200.parallel.fedavg import FedAvgSession, NcclSession  # noqa: E402
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

    def rel(a, b):
        return float((a.double() - b.double()).norm() / b.double().norm().clamp_min(1e-30))

    for kind in ("adam", "yogi"):
        cfg = ServerOptConfig(kind, lr=0.01)
        for wire, nvls in (("fp32", False), ("bf16", False), ("bf16", True), ("fp32", True)):
            arenas = {}
            for name in ("fused", "oracle"):
                torch.manual_seed(0)
                arenas[name] = ParamArena(MLP2(72, 250, 6), dev)
            a_f, a_o = arenas["fused"], arenas["oracle"]
            g_init = a_f.global_w.clone()
            fused = FedAvgSession(a_f, wire_dtype=wire, mode="delta", n_ctas=16, nvls=nvls, server_opt=cfg)
            oracle = NcclSession(a_o, wire_dtype=wire, mode="delta", server_opt=cfg)
            for rnd in range(4):
                # rounds 2 and 3 sample fewer clients than ranks: rank 0 (round 2) or the last rank (round 3) hosts none
                hosts = rnd < 2 or (rank != 0 if rnd == 2 else rank != world - 1)
                n_k = float(1 + rank) if hosts else 0.0
                g = torch.Generator(device=dev).manual_seed(1000 * rnd + rank + 1)
                dl = torch.randn(a_f.n, device=dev, generator=g) * 0.01
                for a in (a_f, a_o):
                    a.theta.copy_(a.global_w + dl)
                fused.aggregate(my_n=n_k)
                oracle.aggregate(my_n=n_k)
                torch.cuda.synchronize(dev)
                fused.check()
                tag = "{} {} nvls={} round {}".format(kind, wire, fused.use_nvls, rnd)
                mf, vf = fused.server_state()
                mo, vo = oracle.server_state()
                expect(rel(a_f.global_w - g_init, a_o.global_w - g_init) < 2e-2, tag + ": fused global_w == oracle")
                expect(rel(mf, mo) < 2e-2 and rel(vf, vo) < 2e-2, tag + ": fused m, v == oracle")
                expect(same_on_every_rank(a_f.global_w) and same_on_every_rank(a_f.theta) and same_on_every_rank(mf)
                       and same_on_every_rank(vf), tag + ": global_w, theta, m, v identical on every rank")
            del fused, oracle
    dist.barrier()
    if rank == 0:
        print("RESULT", "FAIL" if fails else "PASS", len(fails), flush=True)
    dist.destroy_process_group()
    sys.exit(1 if fails else 0)


if __name__ == "__main__":
    main()
