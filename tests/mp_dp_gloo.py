"""CPU / gloo worker for tests/test_dp.py (torchrun --nproc-per-node 2 tests/mp_dp_gloo.py).

Drives :class:`FederatedEngine` with DP-FedAvg through the ``torch.distributed`` session on gloo and checks the global
model after each round against the estimator computed by hand in float64: every rank's delta clipped to ``C``, the
uniform mean over the two participants, plus ``sigma C z(seed, round) / 2``."""
import math
import os
import sys

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from baton_b200.models import MLP2  # noqa: E402
from baton_b200.parallel.dp import normals  # noqa: E402
from baton_b200.parallel.engine import FederatedEngine  # noqa: E402

LR, EPOCHS, C, SIGMA, SEED = 0.05, 2, 0.2, 0.7, 1234


def shard(cid, n):
    g = torch.Generator().manual_seed(3000 + cid)
    X = torch.randn(n, 10, generator=g)
    return X, (X @ torch.arange(1, 11, dtype=torch.float32)).unsqueeze(1) * (1 + cid)


def train_by_hand(params, X, y):
    """Full-batch plain SGD (one batch per epoch, so the sample order does not matter)."""
    params = [p.detach().clone().requires_grad_(True) for p in params]
    for _ in range(EPOCHS):
        h = torch.relu(X @ params[0].t() + params[1])
        loss = torch.nn.functional.mse_loss(h @ params[2].t() + params[3], y)
        grads = torch.autograd.grad(loss, params)
        with torch.no_grad():
            for p, g in zip(params, grads):
                p.sub_(LR * g)
    return [p.detach() for p in params]


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

    sizes = [24 * (r + 1) for r in range(world)]
    X, y = shard(rank, sizes[rank])
    torch.manual_seed(0)
    model = MLP2(10, 16, 1)
    # rank 1 proposes another seed: the engine must use rank 0's on every rank
    eng = FederatedEngine(model, "cpu", backend="nccl", loss="mse", lr=LR, batch_size=sizes[-1], wire_dtype="fp32",
                          name="dp", dp_clip=C, dp_noise_multiplier=SIGMA, dp_seed=SEED if rank == 0 else SEED + 1)
    expect(eng.dp.seed == SEED, "every rank uses rank 0's noise key")
    for rnd in range(2):
        g0 = [p.detach().clone().double() for p in model.parameters()]
        local = train_by_hand(list(model.parameters()), X, y)
        delta = torch.cat([(t.double() - g).flatten() for t, g in zip(local, g0)])
        s = min(1.0, C / float(delta.norm()))
        eng.run_round((X, y), n_epoch=EPOCHS)
        summed = delta * s
        dist.all_reduce(summed)
        n_p = delta.numel()
        z = torch.from_numpy(normals(SEED, rnd, eng.arena.n))[:n_p]
        want = torch.cat([g.flatten() for g in g0]) + (summed + SIGMA * C * z) / world
        got = torch.cat([p.detach().double().flatten() for p in model.parameters()])
        err = float((got - want).abs().max())
        expect(err < 2e-6, "round {}: global model == hand-computed DP-FedAvg (err {:.1e})".format(rnd, err))
        expect(abs(eng.last_clip_factors()[0] - s) < 1e-6 * max(s, 1e-3) and s < 1.0,
               "round {}: clip factor {:.4f} == hand-computed".format(rnd, s))
        expect(torch.equal(eng.arena.theta, eng.arena.global_w), "round {}: theta == global copy".format(rnd))
    eps, _ = eng.privacy_spent(1e-5)
    expect(math.isfinite(eps) and eng.accountant.rounds == 2, "accountant: 2 rounds, epsilon {:.2f}".format(eps))

    dist.barrier()
    if rank == 0:
        print("RESULT", "FAIL" if fails else "PASS", len(fails), flush=True)
    dist.destroy_process_group()
    sys.exit(1 if fails else 0)


if __name__ == "__main__":
    main()
