"""Server-side optimizers (FedAvgM / FedAdagrad / FedYogi / FedAdam) on the flagship configuration: what the step costs
in the collective and per round, and what it does to held-out accuracy on non-IID clients.

* collective: the fused collective alone on ResNet-18's arena (bf16 wire, one CTA per SM, world 1), the plain kernel
  against each kind's *_sopt kernel, blocks alternating between them (median + range).
* round: ResNet-18, 1 GPU, one client, 4096 samples, batch 128, bf16 wire, 256 MiB L2 flush between rounds; engines with
  server_opt off and "adam", blocks of device-timed rounds alternating between them.
* utility: 16 Dirichlet(0.1) clients, 8 per round, 15 rounds, held-out accuracy for FedAvg and each kind at the server
  learning rates in SERVER_LR (b1 = 0.9, b2 = 0.99, tau = 1e-3).  One run per cell.

    python scripts/server_opt_bench.py [--reps 5] [--rounds-per-rep 5] [--parts collective,round] [--skip-utility]

Reads the card name, power limit and SM clock in the same run and prints one JSON line."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from fedprox_bench import card  # noqa: E402
from robust_bench import _alternate  # noqa: E402

KINDS = ("avgm", "adagrad", "yogi", "adam")
SERVER_LR = {"avgm": 1.0, "adagrad": 0.01, "yogi": 0.01, "adam": 0.01}


def collective_cost(args, torch, dev):
    from baton_b200.models import resnet18
    from baton_b200.parallel.arena import ParamArena
    from baton_b200.parallel.fedavg import FedAvgSession
    from baton_b200.parallel.server_opt import ServerOptConfig
    torch.manual_seed(0)
    arena = ParamArena(resnet18(10), dev, momentum=False)
    sms = torch.cuda.get_device_properties(dev).multi_processor_count
    sessions = {}
    for kind in (None,) + KINDS:
        cfg = ServerOptConfig(kind, SERVER_LR[kind]) if kind else None
        sessions[kind or "plain"] = FedAvgSession(arena, wire_dtype="bf16", mode="delta", n_ctas=sms, nvls=False,
                                                  server_opt=cfg)
    # every session allocated its own state: keep each one's (m, v) and point the arena at it before its launches
    state = {name: (arena.server_m, arena.server_v) for name in sessions}
    for name, s in sessions.items():
        if s.server_opt is not None:
            state[name] = s.server_opt.init_state(arena.n_param, dev)

    def time_block(name, k):
        s = sessions[name]
        arena.server_m, arena.server_v = state[name]
        ts = []
        for _ in range(k):
            arena.theta.add_(1e-4)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            s.aggregate(my_n=1.0)
            e1.record()
            e1.synchronize()
            ts.append(e0.elapsed_time(e1) * 1e3)
        s.check()
        return sorted(ts)[len(ts) // 2]
    names = list(sessions)
    for name in names:
        time_block(name, 3)
    got = {name: [] for name in names}
    for r in range(args.reps):
        for name in (names if r % 2 == 0 else names[::-1]):
            got[name].append(time_block(name, 10))
    state_bytes = {name: (0 if sessions[name].server_opt is None else
                          arena.n_param * 4 * (2 if sessions[name].server_opt.needs_v else 1)) for name in names}
    out = {name: {"median_us": sorted(v)[len(v) // 2], "range_us": [min(v), max(v)], "n_param": arena.n_param,
                  "state_bytes": state_bytes[name]} for name, v in got.items()}
    del sessions
    torch.cuda.empty_cache()
    return out


def round_cost(args, torch, dev):
    from baton_b200.data import dirichlet_label_shards, image_shard
    from baton_b200.models import resnet18
    from baton_b200.parallel.engine import FederatedEngine
    X, y = image_shard(dirichlet_label_shards(1, 10, 4096, alpha=0.5, seed=11)[0], seed=3, dtype=torch.bfloat16)
    shard = (X.to(dev), y.to(dev))
    engines = {}
    for name, kw in (("plain", {}), ("adam", {"server_opt": "adam", "server_lr": SERVER_LR["adam"]})):
        torch.manual_seed(0)
        engines[name] = FederatedEngine(resnet18(10), dev, backend="fused", lr=0.05, batch_size=128, n_ctas=132,
                                        seed=5, **kw)

    def run(eng):
        eng.run_round(shard, n_epoch=1, read_loss=False)
        eng.sync()
    out = _alternate(torch, engines, run, args.reps, args.rounds_per_rep)
    for name in engines:
        engines[name].session.check()
    del engines
    torch.cuda.empty_cache()
    return out


def utility(args, torch, dev):
    from baton_b200.data import dirichlet_label_shards, holdout_image_shard, image_shard
    from baton_b200.models import resnet18
    from baton_b200.parallel.engine import FederatedEngine
    n_clients, k = 16, 8
    specs = dirichlet_label_shards(n_clients, 10, args.client_samples, alpha=0.1, seed=11)
    shards = {c: tuple(t.to(dev) for t in image_shard(specs[c], seed=3, dtype=torch.bfloat16)) for c in range(n_clients)}
    Xe, ye = holdout_image_shard(10, 4096, seed=3, dtype=torch.bfloat16)
    held = (Xe.to(dev), ye.to(dev))
    table = {}
    for kind in (None,) + KINDS:
        kw = {"server_opt": kind, "server_lr": SERVER_LR[kind]} if kind else {}
        torch.manual_seed(0)
        eng = FederatedEngine(resnet18(10), dev, backend="fused", lr=0.05, batch_size=128, logical_clients=n_clients,
                              sample_k=k, seed=5, **kw)
        for _ in range(args.utility_rounds):
            eng.run_round(lambda c: shards[c], n_epoch=1, read_loss=False)
        eng.session.check()
        res = eng.evaluate(lambda c: held if c == 0 else None, batch_size=512)
        name = kind or "fedavg"
        table[name] = {"accuracy": round(res.accuracy, 4), "server_lr": SERVER_LR.get(kind)}
        print("utility {:<8} server_lr {} accuracy {:.4f}".format(name, SERVER_LR.get(kind), res.accuracy), flush=True)
        del eng
        torch.cuda.empty_cache()
    return table


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--rounds-per-rep", type=int, default=5)
    ap.add_argument("--parts", default="collective,round")
    ap.add_argument("--skip-utility", action="store_true")
    ap.add_argument("--utility-rounds", type=int, default=15)
    ap.add_argument("--client-samples", type=int, default=512)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("server_opt_bench needs a CUDA device")
    dev = torch.device("cuda:0")
    parts = args.parts.split(",") if args.parts else []
    out = card()
    for name, fn in (("collective", collective_cost), ("round", round_cost)):
        if name in parts:
            out[name] = fn(args, torch, dev)
            print(name, json.dumps(out[name]), flush=True)
    if not args.skip_utility:
        out["utility"] = utility(args, torch, dev)
    out["sm_clock_after"] = card().get("sm_clock")
    print(json.dumps(out))


if __name__ == "__main__":
    main()
