"""FedProx on the flagship configuration: what the proximal term costs, and what it does to a non-IID federation.

* cost: ResNet-18, 1 GPU, 4096 samples, batch 128, bf16, resident shard, 256 MiB L2 flush between rounds (as bench.py
  does).  Blocks of device-timed rounds with prox_mu = 0 and prox_mu = 0.01 alternate on the same engine (both epoch
  graphs are captured during warm-up); per setting the median round time and the range over the blocks.
* effect: 8 logical clients time-sliced on one GPU, Dirichlet alpha = 0.1 label skew, 30 rounds of 2 local epochs,
  the same seeds for every prox_mu in {0, 0.001, 0.01, 0.1}; held-out accuracy of the global model every 5 rounds
  (``FederatedEngine.evaluate`` on ``holdout_image_shard``).

    python scripts/fedprox_bench.py [--reps 7] [--rounds-per-rep 5] [--effect-rounds 30] [--skip-effect]

Reads the card name, power limit and SM clock in the same run and prints one JSON line."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                              "--format=csv,noheader", "-i", "0"],
                             stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True, timeout=30).stdout
        name, power, sm, sm_max = [s.strip() for s in out.strip().splitlines()[0].split(",")]
        return {"card": name, "power_limit": power, "sm_clock": sm, "sm_clock_max": sm_max}
    except Exception:
        import torch
        return {"card": torch.cuda.get_device_name(0), "power_limit": "unknown", "sm_clock": "unknown"}


def cost(args, torch, dev):
    from baton_b200.data import dirichlet_label_shards, image_shard
    from baton_b200.models import resnet18
    from baton_b200.parallel.engine import FederatedEngine
    torch.manual_seed(0)
    eng = FederatedEngine(resnet18(10), dev, backend="fused", lr=0.05, batch_size=128, n_ctas=132, seed=5)
    spec = dirichlet_label_shards(1, 10, 4096, alpha=0.5, seed=11)[0]
    X, y = image_shard(spec, seed=3, dtype=torch.bfloat16)
    shard = (X.to(dev), y.to(dev))
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    mus = (0.0, 0.01)

    def block(mu, k):
        eng.hp["prox_mu"] = mu
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

    for mu in mus:
        block(mu, 3)                                  # capture + warm-up of both epoch graphs
    reps = {mu: [] for mu in mus}
    for r in range(args.reps):
        for mu in (mus if r % 2 == 0 else mus[::-1]):
            reps[mu].append(block(mu, args.rounds_per_rep))
            print("cost rep {} prox_mu={:<5} {:.3f} ms/round".format(r, mu, reps[mu][-1]), flush=True)
    out = {"graphs": len(eng.trainer._graphs)}
    for mu, v in reps.items():
        out["round_ms_mu{}".format(mu)] = sorted(v)[len(v) // 2]
        out["round_ms_range_mu{}".format(mu)] = [min(v), max(v)]
    out["overhead"] = out["round_ms_mu0.01"] / out["round_ms_mu0.0"] - 1.0
    return out


def effect(args, torch, dev):
    from baton_b200.data import dirichlet_label_shards, holdout_image_shard, image_shard
    from baton_b200.models import resnet18
    from baton_b200.parallel.engine import FederatedEngine
    n_clients = 8
    specs = dirichlet_label_shards(n_clients, 10, args.client_samples, alpha=0.1, seed=11)
    shards = {c: tuple(t.to(dev) for t in image_shard(specs[c], seed=3, dtype=torch.bfloat16)) for c in range(n_clients)}
    Xe, ye = holdout_image_shard(10, 4096, seed=3, dtype=torch.bfloat16)
    held = (Xe.to(dev), ye.to(dev))
    curves = {}
    for mu in (0.0, 0.001, 0.01, 0.1):
        torch.manual_seed(0)
        eng = FederatedEngine(resnet18(10), dev, backend="fused", lr=0.05, batch_size=128, logical_clients=n_clients,
                              seed=5, prox_mu=mu)
        acc = []
        for rnd in range(1, args.effect_rounds + 1):
            eng.run_round(lambda c: shards[c], n_epoch=2, read_loss=False)
            if rnd % 5 == 0:
                res = eng.evaluate(lambda c: held if c == 0 else None, batch_size=512)
                acc.append(round(res.accuracy, 4))
                print("effect prox_mu={:<5} round {:2d} held-out accuracy {:.4f}".format(mu, rnd, res.accuracy),
                      flush=True)
        curves[str(mu)] = acc
        del eng
        torch.cuda.empty_cache()
    return {"clients": n_clients, "client_samples": args.client_samples, "alpha": 0.1, "local_epochs": 2,
            "rounds": args.effect_rounds, "eval_every": 5, "heldout_accuracy": curves}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--rounds-per-rep", type=int, default=5)
    ap.add_argument("--effect-rounds", type=int, default=30)
    ap.add_argument("--client-samples", type=int, default=1024)
    ap.add_argument("--skip-effect", action="store_true")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("fedprox_bench.py measures on a CUDA device; none is available")
    dev = torch.device("cuda:0")
    out = card()
    out["cost"] = cost(args, torch, dev)
    if not args.skip_effect:
        out["effect"] = effect(args, torch, dev)
    out["sm_clock_after"] = card().get("sm_clock")
    print(json.dumps(out))


if __name__ == "__main__":
    main()
