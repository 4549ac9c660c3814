"""SCAFFOLD on the flagship configuration: what the control variates cost per round, and what they do to a non-IID
federation.

* cost: ResNet-18, 1 GPU, 4096 samples, batch 128, bf16, resident shard, 256 MiB L2 flush between rounds (as bench.py
  does).  Two engines, scaffold=False and scaffold=True, run alternating blocks of device-timed rounds (both epoch
  graphs are captured during warm-up); per setting the median round time and the range over the blocks.
* utility: 64 logical clients time-sliced on one GPU, Dirichlet alpha = 0.1 label skew, 16 clients sampled per round,
  the same seeds for FedAvg, FedProx (prox_mu = 0.01) and SCAFFOLD; held-out accuracy of the global model every 5
  rounds (``FederatedEngine.evaluate`` on ``holdout_image_shard``).

    python scripts/scaffold_bench.py [--reps 7] [--rounds-per-rep 5] [--effect-rounds 20] [--skip-effect]

Reads the card name, power limit and SM clock in the same run and prints one JSON line."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from fedprox_bench import card  # noqa: E402


def cost(args, torch, dev):
    from baton_b200.data import dirichlet_label_shards, image_shard
    from baton_b200.models import resnet18
    from baton_b200.parallel.engine import FederatedEngine
    spec = dirichlet_label_shards(1, 10, 4096, alpha=0.5, seed=11)[0]
    X, y = image_shard(spec, seed=3, dtype=torch.bfloat16)
    shard = (X.to(dev), y.to(dev))
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    engines = {}
    for on in (False, True):
        torch.manual_seed(0)
        engines[on] = FederatedEngine(resnet18(10), dev, backend="fused", lr=0.05, batch_size=128, n_ctas=132, seed=5,
                                      scaffold=on)

    def block(on, k):
        eng = engines[on]
        ms = []
        for _ in range(k):
            flush.zero_()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            eng.run_round(shard, n_epoch=1, read_loss=False)
            eng.sync()
            e1.record()
            e1.synchronize()
            ms.append(e0.elapsed_time(e1))
        return sorted(ms)[len(ms) // 2]

    for on in (False, True):
        block(on, 3)                                  # capture + warm-up
    reps = {on: [] for on in (False, True)}
    for r in range(args.reps):
        for on in ((False, True) if r % 2 == 0 else (True, False)):
            reps[on].append(block(on, args.rounds_per_rep))
            print("cost rep {} scaffold={!s:<5} {:.3f} ms/round".format(r, on, reps[on][-1]), flush=True)
    out = {}
    for on, v in reps.items():
        key = "on" if on else "off"
        out["round_ms_" + key] = sorted(v)[len(v) // 2]
        out["round_ms_range_" + key] = [min(v), max(v)]
    out["overhead"] = out["round_ms_on"] / out["round_ms_off"] - 1.0
    out["wire_bytes"] = {"off": engines[False].session.wire_bytes(), "on": engines[True].session.wire_bytes()}
    return out


def effect(args, torch, dev):
    from baton_b200.data import dirichlet_label_shards, holdout_image_shard, image_shard
    from baton_b200.models import resnet18
    from baton_b200.parallel.engine import FederatedEngine
    n_clients, k = 64, 16
    specs = dirichlet_label_shards(n_clients, 10, args.client_samples, alpha=0.1, seed=11)
    shards = {c: tuple(t.to(dev) for t in image_shard(specs[c], seed=3, dtype=torch.bfloat16)) for c in range(n_clients)}
    Xe, ye = holdout_image_shard(10, 4096, seed=3, dtype=torch.bfloat16)
    held = (Xe.to(dev), ye.to(dev))
    curves = {}
    for name, kw in (("fedavg", {}), ("fedprox_0.01", {"prox_mu": 0.01}), ("scaffold", {"scaffold": True})):
        torch.manual_seed(0)
        eng = FederatedEngine(resnet18(10), dev, backend="fused", lr=0.05, batch_size=128, logical_clients=n_clients,
                              sample_k=k, seed=5, **kw)
        acc = []
        for rnd in range(1, args.effect_rounds + 1):
            eng.run_round(lambda c: shards[c], n_epoch=args.local_epochs, read_loss=False)
            if rnd % 5 == 0:
                res = eng.evaluate(lambda c: held if c == 0 else None, batch_size=512)
                acc.append(round(res.accuracy, 4))
                print("effect {:<12} round {:2d} held-out accuracy {:.4f}".format(name, rnd, res.accuracy), flush=True)
        curves[name] = acc
        del eng
        torch.cuda.empty_cache()
    return {"clients": n_clients, "sampled": k, "client_samples": args.client_samples, "alpha": 0.1,
            "local_epochs": args.local_epochs, "rounds": args.effect_rounds, "eval_every": 5,
            "heldout_accuracy": curves}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--rounds-per-rep", type=int, default=5)
    ap.add_argument("--effect-rounds", type=int, default=20)
    ap.add_argument("--client-samples", type=int, default=512)
    ap.add_argument("--local-epochs", type=int, default=2)
    ap.add_argument("--skip-effect", action="store_true")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("scaffold_bench.py measures on a CUDA device; none is available")
    dev = torch.device("cuda:0")
    out = card()
    out["cost"] = cost(args, torch, dev)
    if not args.skip_effect:
        out["effect"] = effect(args, torch, dev)
    out["sm_clock_after"] = card().get("sm_clock")
    print(json.dumps(out))


if __name__ == "__main__":
    main()
