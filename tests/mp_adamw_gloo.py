"""Local AdamW across two gloo ranks (torchrun --nproc-per-node 2 tests/mp_adamw_gloo.py), and the hand-written
"fresh AdamW per client per round, then the FedAvg mean" that tests/test_adamw.py also checks the one-rank engine
against.

Every client trains full-batch (one step per epoch, so the sample order does not matter) with the AdamW of
``torch.optim.AdamW`` written out: decoupled weight decay, then the bias-corrected moment step, ``t`` counting across
the epochs of the client's run and the moments starting at zero in every round."""
import math
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from mp_scaffold_gloo import _mlp_loss, shard  # noqa: E402

LR, EPOCHS, WD, BETAS, EPS = 0.01, 3, 0.05, (0.8, 0.99), 1e-6


def adamw_by_hand(init, rounds, shards):
    """Global model after ``rounds`` (lists of participating client ids)."""
    b1, b2 = BETAS
    x = [p.clone().double() for p in init]
    for part in rounds:
        models, weights = [], []
        for cid in part:
            X, y = (t.double() for t in shards(cid))
            params = [p.clone().requires_grad_(True) for p in x]
            m = [torch.zeros_like(p) for p in x]
            v = [torch.zeros_like(p) for p in x]
            for t in range(1, EPOCHS + 1):
                grads = torch.autograd.grad(_mlp_loss(params, X, y), params)
                with torch.no_grad():
                    for p, g, mk, vk in zip(params, grads, m, v):
                        p.mul_(1 - LR * WD)
                        mk.mul_(b1).add_((1 - b1) * g)
                        vk.mul_(b2).add_((1 - b2) * g * g)
                        p.sub_(LR / (1 - b1 ** t) * mk / (vk.sqrt() / math.sqrt(1 - b2 ** t) + EPS))
            models.append([p.detach() for p in params])
            weights.append(float(X.shape[0]))
        tot = sum(weights)
        x = [xp + sum(w * (mo[k] - xp) for w, mo in zip(weights, models)) / tot for k, xp in enumerate(x)]
    return x


def global_error(eng, init, rounds, shards):
    """Max abs error of the engine's global model against :func:`adamw_by_hand`, relative to its largest magnitude."""
    want = adamw_by_hand(init, rounds, shards)
    a = eng.arena
    names = [n for n, _ in eng.model.named_parameters()]
    scale = max(float(w.abs().max()) for w in want)
    return max(float((a._view(a.global_w, a.slots[n]).double() - w).abs().max()) for n, w in zip(names, want)) / scale


def make_engine(n_clients, sample_k, seed, **kw):
    from baton_b200.models import MLP2
    from baton_b200.parallel.engine import FederatedEngine
    torch.manual_seed(0)
    model = MLP2(10, 16, 1)
    init = [p.detach().clone() for p in model.parameters()]
    eng = FederatedEngine(model, "cpu", backend="nccl", loss="mse", lr=LR, batch_size=64, wire_dtype="fp32",
                          weight_decay=WD, optimizer="adamw", betas=BETAS, eps=EPS, logical_clients=n_clients,
                          sample_k=sample_k, seed=seed, **kw)
    return eng, init


def main():
    import torch.distributed as dist
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

    sizes = lambda cid: 16 + 4 * cid                               # noqa: E731
    eng, init = make_engine(6, 3, 5)
    rounds = [eng.run_round(lambda cid: shard(cid, sizes(cid)), n_epoch=EPOCHS).participants for _ in range(3)]
    err = global_error(eng, init, rounds, lambda cid: shard(cid, sizes(cid)))
    expect(err < 2e-5, "engine == hand-written local AdamW + FedAvg on rank {} ({:.1e})".format(rank, err))
    g0 = eng.arena.global_w.clone()
    dist.broadcast(g0, 0)
    expect(torch.equal(eng.arena.global_w, g0), "the global model is identical on every rank")

    dist.barrier()
    if rank == 0:
        print("RESULT", "FAIL" if fails else "PASS", len(fails), flush=True)
    dist.destroy_process_group()
    sys.exit(1 if fails else 0)


if __name__ == "__main__":
    main()
