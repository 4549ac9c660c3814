"""Personalized FL (FedBN / FedPer, ``local_keys``) on the flagship configuration: what the compact wire and the lost
optimizer-emitted upload cost, and what personalization does to each client's held-out accuracy.

* collective: the fused collective alone on ResNet-18's arena (bf16 wire, one CTA per SM, world 1): the plain kernel
  against the personalized kernel with the FedBN and the FedPer range, blocks alternating between them (median + range).
* round: ResNet-18, 1 GPU, one client, 4096 samples, batch 128, bf16 wire, 256 MiB L2 flush between rounds; engines with
  local_keys None and "bn", blocks of device-timed rounds alternating between them.
* utility: 16 Dirichlet(0.1) clients of 512 samples, 8 per round, 15 rounds; the mean over clients of the accuracy on
  each client's own held-out samples (client_holdout_image_shard) with its personalized model, for FedAvg, FedBN, FedPer
  and FedBN + FedPer, at shift 0 and at --shift.  One run per cell.

    python scripts/personal_bench.py [--reps 5] [--rounds-per-rep 5] [--parts collective,round] [--skip-utility]

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

METHODS = {"fedavg": None, "fedbn": "bn", "fedper": "head", "fedbn+fedper": ("bn", "head")}


def collective_cost(args, torch, dev):
    from baton_b200.models import resnet18
    from baton_b200.parallel.arena import ParamArena
    from baton_b200.parallel.fedavg import FedAvgSession
    from baton_b200.parallel.personal import resolve_local_keys
    sms = torch.cuda.get_device_properties(dev).multi_processor_count
    sessions, arenas = {}, {}
    for name in ("plain", "fedbn", "fedper"):
        torch.manual_seed(0)
        m = resnet18(10)
        keys = resolve_local_keys(m, METHODS[name]) if name != "plain" else ()
        arenas[name] = ParamArena(m, dev, momentum=False, local=keys)
        sessions[name] = FedAvgSession(arenas[name], wire_dtype="bf16", mode="delta", n_ctas=sms, nvls=False,
                                       local=bool(keys))

    def time_block(name, k):
        s, a = sessions[name], arenas[name]
        ts = []
        for _ in range(k):
            a.theta.add_(1e-4)
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
    out = {name: {"median_us": sorted(v)[len(v) // 2], "range_us": [min(v), max(v)], "n": arenas[name].n,
                  "n_wire": arenas[name].n_shared, "wire_bytes": sessions[name].wire_bytes()} for name, v in got.items()}
    del sessions, arenas
    torch.cuda.empty_cache()
    return out


def round_cost(args, torch, dev):
    from baton_b200.data import dirichlet_label_shards, image_shard
    from baton_b200.models import resnet18
    from baton_b200.parallel.engine import FederatedEngine
    X, y = image_shard(dirichlet_label_shards(1, 10, 4096, alpha=0.5, seed=11)[0], seed=3, dtype=torch.bfloat16)
    shard = (X.to(dev), y.to(dev))
    engines = {}
    for name, lk in (("plain", None), ("fedbn", "bn")):
        torch.manual_seed(0)
        engines[name] = FederatedEngine(resnet18(10), dev, backend="fused", lr=0.05, batch_size=128, n_ctas=132,
                                        seed=5, local_keys=lk)

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
    from baton_b200.data import client_holdout_image_shard, dirichlet_label_shards, image_shard
    from baton_b200.models import resnet18
    from baton_b200.parallel.engine import FederatedEngine
    n_clients, k = 16, 8
    specs = dirichlet_label_shards(n_clients, 10, args.client_samples, alpha=0.1, seed=11)
    table = {}
    for shift in (0.0, args.shift):
        shards = {c: tuple(t.to(dev) for t in image_shard(specs[c], seed=3, dtype=torch.bfloat16, shift=shift))
                  for c in range(n_clients)}
        held = {c: tuple(t.to(dev) for t in client_holdout_image_shard(specs[c], 256, seed=3, dtype=torch.bfloat16,
                                                                         shift=shift)) for c in range(n_clients)}
        for name, lk in METHODS.items():
            torch.manual_seed(0)
            eng = FederatedEngine(resnet18(10), dev, backend="fused", lr=0.05, batch_size=128,
                                  logical_clients=n_clients, sample_k=k, seed=5, local_keys=lk)
            for _ in range(args.utility_rounds):
                eng.run_round(lambda c: shards[c], n_epoch=1, read_loss=False)
            eng.session.check()
            accs = [eng.evaluate(lambda cid, c=c: held[c] if cid == c else None, batch_size=256).local_accuracy
                    for c in range(n_clients)]
            mean = sum(accs) / len(accs)
            table["{}@shift={}".format(name, shift)] = {"mean_client_accuracy": round(mean, 4),
                                                       "min": round(min(accs), 4), "max": round(max(accs), 4)}
            print("utility {:<13} shift {} mean personalized accuracy {:.4f}".format(name, shift, mean), flush=True)
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
    ap.add_argument("--shift", type=float, default=0.5)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("personal_bench needs a CUDA device")
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
