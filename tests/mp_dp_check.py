"""Multi-rank worker for tests/test_gpu_dp.py (torchrun --nproc-per-node N tests/mp_dp_check.py, N >= 2).

The fused DP-FedAvg collective against the ``NcclSession`` oracle at the same seed: every rank's clip factor is read by
its peers from the peer-mapped clip pages (double-buffered by round parity: several rounds in a row), the clients per
rank ride on the barrier flags, a rank left out of the alive mask, and a rank whose update is not finite (s = 0: the
readers skip its wire, the global model stays finite on every replica)."""
import math
import os
import sys

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from baton_b200.models import MLP2  # noqa: E402
from baton_b200.parallel.arena import ParamArena  # noqa: E402
from baton_b200.parallel.dp import DPConfig  # noqa: E402
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

    arenas = {}
    for name in ("fused", "oracle"):
        torch.manual_seed(0)
        arenas[name] = ParamArena(MLP2(72, 250, 6), dev, momentum=True)
    a_f, a_o = arenas["fused"], arenas["oracle"]
    # rank 1 proposes another key: both sessions must take rank 0's
    dp = DPConfig(0.05, 1.0, seed=4242 if rank == 0 else 99)
    fused = FedAvgSession(a_f, wire_dtype="fp32", mode="delta", n_ctas=16, dp=dp)
    oracle = NcclSession(a_o, wire_dtype="fp32", mode="delta", dp=dp)
    expect(fused.dp.seed == 4242 and oracle.dp.seed == 4242, "every rank uses rank 0's noise key")
    expect(not fused.use_nvls, "DP sessions run on peer loads")

    def drift(rnd, scale):
        g = torch.Generator(device=dev).manual_seed(1000 * rnd + rank)
        d = torch.randn(a_f.n, device=dev, generator=g) * scale
        for a in (a_f, a_o):
            a.theta.copy_(a.global_w + d)

    def compare(tag, ranks):
        err = float((a_f.global_w - a_o.global_w).abs().max()) if rank in ranks else 0.0
        expect(err < 1e-6, "{}: fused == NCCL oracle (max err {:.1e})".format(tag, err))
        ref = a_f.global_w.clone()
        dist.broadcast(ref, src=0)
        same = torch.equal(a_f.global_w, ref) if rank in ranks else True
        expect(same, "{}: every live replica holds the same global model".format(tag))

    # several rounds with counts on the barrier flags: the clip pages alternate halves
    for rnd in range(3):
        drift(rnd, 0.002 * (rank + 1))
        fused.aggregate(my_n=1.0)
        oracle.aggregate(my_n=1.0)
        torch.cuda.synchronize()
        fused.check()
        s_f, s_o = fused.last_clip_factors()[0], oracle.last_clip_factors()[0]
        expect(abs(s_f - s_o) <= 1e-5 * s_o and s_o < 1.0, "round {}: clip factor {:.4f} == oracle".format(rnd, s_o))
        compare("round {} (flags)".format(rnd), range(world))

    # the last rank is not alive: neither read, written nor waited for; the host plan carries the clients per rank
    drift(3, 0.003)
    last = world - 1
    counts = [1.0] * (world - 1) + [0.0]
    fused.aggregate(n_samples_by_rank=counts, alive_ranks=list(range(world - 1)))
    oracle.aggregate(n_samples_by_rank=counts)
    torch.cuda.synchronize()
    fused.check()
    compare("alive mask without rank {}".format(last), range(world - 1))
    expect(fused.stale if rank == last else not fused.stale, "the excluded rank knows its replica is stale")
    for a in (a_f, a_o):                      # bring the excluded replica back to the global model
        dist.broadcast(a.global_w, src=0)
        a.theta.copy_(a.global_w)

    # rank 0 uploads a non-finite update: s_0 = 0, it still counts in m, nobody reads its wire
    drift(4, 0.002)
    if rank == 0:
        for a in (a_f, a_o):
            a.theta[5] = float("nan")
            a.theta[7] = float("inf")
    bad_before = fused.nonfinite_updates()
    fused.aggregate(my_n=1.0)
    oracle.aggregate(my_n=1.0)
    torch.cuda.synchronize()
    fused.check()
    expect(bool(torch.isfinite(a_f.global_w).all()), "a non-finite upload does not poison the global model")
    expect((fused.last_clip_factors()[0] == 0.0) == (rank == 0) and
           fused.nonfinite_updates() - bad_before == (1 if rank == 0 else 0),
           "the non-finite update gets s = 0 and is counted")
    compare("non-finite upload on rank 0", range(world))
    expect(math.isfinite(float(a_f.global_w.abs().max())), "finite after the poisoned round")

    dist.barrier()
    if rank == 0:
        print("RESULT", "FAIL" if fails else "PASS", len(fails), flush=True)
    dist.destroy_process_group()
    sys.exit(1 if fails else 0)


if __name__ == "__main__":
    main()
