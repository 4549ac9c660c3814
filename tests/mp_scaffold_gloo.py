"""SCAFFOLD across two gloo ranks (torchrun --nproc-per-node 2 tests/mp_scaffold_gloo.py), and the hand-written
SCAFFOLD that tests/test_scaffold.py also checks the one-rank engine against.

Every client trains full-batch (one step per epoch, so the sample order does not matter) with
``w -= lr * (g + c - c_i)``; then ``dc_i = (x - y_i) / (K lr) - c``, ``c_i += dc_i``, the global model becomes the
sample-weighted mean of the clients' models and ``c += sum(dc_i) / N``."""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

LR, EPOCHS = 0.01, 3


def shard(cid, n):
    g = torch.Generator().manual_seed(3000 + cid)
    X = torch.randn(n, 10, generator=g)
    w = torch.arange(1, 11, dtype=torch.float32) * (1.0 + 0.3 * cid)        # non-IID targets
    return X, (X @ w).unsqueeze(1) + 0.01 * torch.randn(n, 1, generator=g)


def _mlp_loss(params, X, y):
    h = torch.relu(X @ params[0].t() + params[1])
    return torch.nn.functional.mse_loss(h @ params[2].t() + params[3], y)


def scaffold_by_hand(init, rounds, shards, n_clients):
    """Global model, c and every c_i after ``rounds`` (lists of participating client ids)."""
    x = [p.clone() for p in init]
    c = [torch.zeros_like(p) for p in init]
    ci = {}
    for part in rounds:
        models, weights, dcs = [], [], []
        for cid in part:
            X, y = shards(cid)
            cv = ci.setdefault(cid, [torch.zeros_like(p) for p in init])
            params = [p.clone().requires_grad_(True) for p in x]
            for _ in range(EPOCHS):
                grads = torch.autograd.grad(_mlp_loss(params, X, y), params)
                with torch.no_grad():
                    for p, g, a, b in zip(params, grads, c, cv):
                        p.sub_(LR * (g + a - b))
            yi = [p.detach() for p in params]
            dc = [(a - b) / (EPOCHS * LR) - cc for a, b, cc in zip(x, yi, c)]
            ci[cid] = [a + d for a, d in zip(cv, dc)]
            models.append(yi)
            weights.append(float(X.shape[0]))
            dcs.append(dc)
        tot = sum(weights)
        x = [xp + sum(w * (m[k] - xp) for w, m in zip(weights, models)) / tot for k, xp in enumerate(x)]
        c = [cp + sum(d[k] for d in dcs) / n_clients for k, cp in enumerate(c)]
    return x, c, ci


def check_against_hand_written(eng, init, rounds, shards, n_clients, hosted):
    """Max abs errors, relative to the largest magnitude of each reference, of the engine's global model, c and hosted
    c_i against :func:`scaffold_by_hand` (dc divides a model difference by K lr, which scales its rounding too)."""
    x, c, ci = scaffold_by_hand(init, rounds, shards, n_clients)
    a = eng.arena
    names = [n for n, _ in eng.model.named_parameters()]
    got_c, got_ci = eng.control_variates()

    def err(flat, want):
        scale = max(float(w.abs().max()) for w in want) + 1e-12
        return max(float((a._view(flat, a.slots[n]) - w).abs().max()) for n, w in zip(names, want)) / scale
    out = {"global": err(a.global_w, x), "c": err(got_c, c)}
    for cid, want in ci.items():
        if hosted(cid):
            out["c_{}".format(cid)] = err(got_ci[cid], want)
    return out


def main():
    import torch.distributed as dist
    from baton_b200.models import MLP2
    from baton_b200.parallel.engine import FederatedEngine
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

    n_clients = 6
    sizes = lambda cid: 16 + 4 * cid                               # noqa: E731
    torch.manual_seed(0)
    model = MLP2(10, 16, 1)
    init = [p.detach().clone() for p in model.parameters()]
    eng = FederatedEngine(model, "cpu", backend="nccl", loss="mse", lr=LR, batch_size=64, wire_dtype="fp32",
                          scaffold=True, logical_clients=n_clients, sample_k=3, seed=5)
    rounds = [eng.run_round(lambda cid: shard(cid, sizes(cid)), n_epoch=EPOCHS).participants for _ in range(3)]
    errs = check_against_hand_written(eng, init, rounds, lambda cid: shard(cid, sizes(cid)), n_clients,
                                      hosted=eng.hosted)
    expect(max(errs.values()) < 2e-5, "engine == hand-written SCAFFOLD on rank {} ({})".format(
        rank, ", ".join("{} {:.1e}".format(k, v) for k, v in sorted(errs.items()))))
    c, _ = eng.control_variates()
    c0 = c.clone()
    dist.broadcast(c0, 0)
    expect(torch.equal(c, c0), "c is identical on every rank")
    expect(torch.equal(eng.arena.theta, eng.arena.global_w), "theta == global copy after the round")

    dist.barrier()
    if rank == 0:
        print("RESULT", "FAIL" if fails else "PASS", len(fails), flush=True)
    dist.destroy_process_group()
    sys.exit(1 if fails else 0)


if __name__ == "__main__":
    main()
