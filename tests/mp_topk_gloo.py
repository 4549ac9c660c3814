"""CPU / gloo worker for tests/test_topk.py (torchrun --nproc-per-node 2 tests/mp_topk_gloo.py).

Two ranks run a FederatedEngine (backend='nccl') with top-k 10 % uploads, error feedback and FedAvgM on 6 logical
clients, 3 sampled per round, for 4 rounds.  Local training is replaced by a known update per (client, round), so a
closed-form host replay of the rule follows the engine: a rank with one hosted participant uploads its topk(u); a rank
with several folds n_k * topk(u_k) and uploads the folded mean; the server adds the sample-weighted uploads and steps
FedAvgM.  After every round the global model must equal the replay bit for bit on both ranks, the residuals of the
clients a rank hosts must equal the replay's (a client that sat out keeps its residual), and only clients that took
part have one."""
import os
import random
import sys

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from baton_b200.models import MLP2  # noqa: E402
from baton_b200.parallel.compress import TopKConfig, n_float, topk_select  # noqa: E402
from baton_b200.parallel.engine import FederatedEngine  # noqa: E402
from baton_b200.parallel.server_opt import ServerOptConfig, apply_update_  # noqa: E402

CLIENTS, SAMPLE, ROUNDS, SEED, RATIO = 6, 3, 4, 11, 0.1


def _delta(n, cid, rnd):
    return torch.randn(n, generator=torch.Generator().manual_seed(1000 * rnd + cid)) * 0.01


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

    torch.manual_seed(0)
    eng = FederatedEngine(MLP2(10, 64, 3), "cpu", backend="nccl", wire_dtype="fp32", logical_clients=CLIENTS,
                          sample_k=SAMPLE, seed=SEED, compress="topk", topk_ratio=RATIO, server_opt="avgm",
                          server_lr=1.0)
    a = eng.arena
    mask = torch.zeros(a.n)
    for s in a.slots.values():      # training never moves the alignment padding
        mask[s.offset: s.offset + s.numel] = 1.0

    def fake_run(X, y, n_epoch=1, **_kw):
        a.theta.copy_(a.global_w + _delta(a.n, int(X[0, 0]), eng.n_rounds) * mask)
        return torch.zeros(n_epoch, 2)
    eng.trainer.run = fake_run
    eng.trainer.last_steps = 1
    shards = lambda c: (torch.full((4 + c, 10), float(c)), torch.zeros(4 + c, dtype=torch.long))   # noqa: E731

    k = TopKConfig(RATIO).k(n_float(a))
    cfg = ServerOptConfig("avgm", 1.0)
    x = a.global_w.clone()
    m, v = cfg.init_state(a.n_param, "cpu")
    res = {}
    rng = random.Random(SEED)
    for rnd in range(ROUNDS):
        eng.run_round(shards)
        parts = sorted(rng.sample(range(CLIENTS), SAMPLE))
        counts = torch.tensor([float(sum(4 + c for c in parts if c % world == r)) for r in range(world)])
        total = counts.sum()
        d = torch.zeros(a.n)
        for r in range(world):
            mine = [c for c in parts if c % world == r]
            ups = []
            for c in mine:
                e = res.setdefault(c, torch.zeros(a.n))
                th = x + _delta(a.n, c, rnd) * mask
                u = (th - x) + e
                idx = topk_select(u, k)
                top = torch.zeros(a.n)
                top[idx] = u[idx]
                e.copy_(u)
                e[idx] = 0.0
                ups.append((4 + c, idx, u[idx]))
            if not mine:
                continue
            if len(mine) == 1:
                up = torch.zeros(a.n)
                up[ups[0][1]] = ups[0][2]
            else:
                acc = torch.zeros(a.n)
                for nk, idx, vals in ups:
                    acc[idx] += vals * float(nk)
                up = torch.add(x, acc, alpha=1.0 / float(counts[r])) - x
            d = d + (up * (counts[r] / total)).to(torch.float32)
        apply_update_(x, d, a.n_param, m, v, cfg)
        tag = "round {} ({})".format(rnd, parts)
        expect(torch.equal(a.global_w.view(torch.int32), x.view(torch.int32)), tag + ": global model = host replay")
        mine_res = eng.topk_residuals()
        hosted = {c: e for c, e in res.items() if c % world == rank}
        expect(set(mine_res) == set(hosted), tag + ": residuals exactly for the hosted clients that took part")
        expect(all(torch.equal(mine_res[c], hosted[c]) for c in hosted), tag + ": residuals = host replay")
        entries = eng.session.last_upload_entries()
        mine = [c for c in parts if c % world == rank]
        expect((entries == 0) == (not mine) and entries <= len(mine) * k, tag + ": upload entry count")
    dist.barrier()
    if rank == 0:
        print("RESULT", "FAIL" if fails else "PASS", len(fails), flush=True)
    dist.destroy_process_group()
    sys.exit(1 if fails else 0)


if __name__ == "__main__":
    main()
