"""Multi-rank worker for tests/test_gpu_scaffold.py (torchrun --nproc-per-node N tests/mp_scaffold_check.py, N >= 2).

The fused SCAFFOLD collective against the ``NcclSession`` oracle over several rounds (both wire halves): the model
segment and the control-variate segment, a round in which rank 1 has no participant (its dc must not be read), and
every wire format's own tolerance."""
import os
import sys

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from baton_b200.models import MLP2  # noqa: E402
from baton_b200.parallel.arena import ParamArena  # noqa: E402
from baton_b200.parallel.fedavg import FedAvgSession, NcclSession  # noqa: E402


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

    n_clients = 3 * world
    for wire, tol in (("fp32", 1e-6), ("bf16", 2e-2), ("fp8", 1.5e-1)):
        arenas = {}
        for name in ("fused", "oracle"):
            torch.manual_seed(0)
            arenas[name] = ParamArena(MLP2(72, 250, 6), dev)
        a_f, a_o = arenas["fused"], arenas["oracle"]
        fused = FedAvgSession(a_f, wire_dtype=wire, mode="delta", n_ctas=16, scaffold=True)
        oracle = NcclSession(a_o, wire_dtype="fp32", mode="delta", scaffold=True)
        expect(not fused.use_nvls, "{}: SCAFFOLD sessions run on peer loads".format(wire))
        n_p = a_f.n_param
        c_f, c_o = torch.zeros(n_p, device=dev), torch.zeros(n_p, device=dev)
        gen = torch.Generator(device=dev).manual_seed(100 + rank)
        for rnd in range(4):
            step = torch.randn(a_f.n, device=dev, generator=gen) * 0.01
            dc = torch.randn(n_p, device=dev, generator=gen)
            my_n = 0.0 if (rnd == 2 and rank == 1) else float(32 + 8 * rank)
            if my_n == 0.0:
                dc.fill_(float("nan"))              # a rank without participants: its upload must not be read
                step.zero_()
            for a in (a_f, a_o):
                a.theta.add_(step)
            fused.aggregate(my_n=my_n, control=(c_f, dc, n_clients))
            oracle.aggregate(my_n=my_n, control=(c_o, dc, n_clients))
            torch.cuda.synchronize(dev)
            fused.check()
        gerr = float((a_f.global_w - a_o.global_w).abs().max() / a_o.global_w.abs().max())
        cerr = float((c_f - c_o).abs().max() / c_o.abs().max())
        expect(gerr < tol and torch.isfinite(a_f.global_w).all(), "{}: global model == NCCL oracle ({:.1e})".format(
            wire, gerr))
        expect(cerr < tol and torch.isfinite(c_f).all(), "{}: c == NCCL oracle ({:.1e})".format(wire, cerr))
        ref = c_f.clone()
        dist.broadcast(ref, 0)
        expect(torch.equal(ref, c_f), "{}: c is identical on every rank".format(wire))

    dist.barrier()
    if rank == 0:
        print("RESULT", "FAIL" if fails else "PASS", len(fails), flush=True)
    dist.destroy_process_group()
    sys.exit(1 if fails else 0)


if __name__ == "__main__":
    main()
