"""DP-FedAvg on the flagship configuration: what clipping + noise cost per round, and what they do to accuracy.

* cost: ResNet-18, 1 GPU, 4096 samples, batch 128, bf16, resident shard, 256 MiB L2 flush between rounds (as bench.py
  does).  Two engines with the same model and data, DP off and DP on (C = 1, sigma = 1); blocks of device-timed rounds
  alternate between them.  Per setting the median round time and the range over the blocks.
* utility: 64 logical clients on one GPU, 16 sampled per round, Dirichlet alpha = 0.5 label skew, R rounds of one local
  epoch, the same seeds for every sigma in {0, 0.5, 1}; held-out accuracy of the global model and the
  (epsilon, delta = 1e-5) of the RDP accountant after R rounds.  C is ``--clip``, by default the median update norm of
  the clients of one warm-up round (so about half the updates are clipped).

    python scripts/dp_bench.py [--reps 7] [--rounds-per-rep 5] [--utility-rounds 20] [--clip C] [--skip-utility]

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
    engines = {}
    for name, kw in (("off", {}), ("on", {"dp_clip": 1.0, "dp_noise_multiplier": 1.0})):
        torch.manual_seed(0)
        engines[name] = FederatedEngine(resnet18(10), dev, backend="fused", lr=0.05, batch_size=128, n_ctas=132,
                                        seed=5, **kw)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)

    def block(name, k):
        eng = engines[name]
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
    for name in engines:
        block(name, 3)                                # capture + warm-up
    reps = {name: [] for name in engines}
    for r in range(args.reps):
        for name in (("off", "on") if r % 2 == 0 else ("on", "off")):
            reps[name].append(block(name, args.rounds_per_rep))
            print("cost rep {} dp={:<3} {:.3f} ms/round".format(r, name, reps[name][-1]), flush=True)
    out = {}
    for name, v in reps.items():
        out["round_ms_dp_" + name] = sorted(v)[len(v) // 2]
        out["round_ms_range_dp_" + name] = [min(v), max(v)]
    out["overhead"] = out["round_ms_dp_on"] / out["round_ms_dp_off"] - 1.0
    return out


def utility(args, torch, dev):
    from baton_b200.data import dirichlet_label_shards, holdout_image_shard, image_shard
    from baton_b200.models import resnet18
    from baton_b200.parallel.engine import FederatedEngine
    n_clients, k = 64, 16
    specs = dirichlet_label_shards(n_clients, 10, args.client_samples, alpha=0.5, seed=11)
    shards = {c: tuple(t.to(dev) for t in image_shard(specs[c], seed=3, dtype=torch.bfloat16)) for c in range(n_clients)}
    Xe, ye = holdout_image_shard(10, 4096, seed=3, dtype=torch.bfloat16)
    held = (Xe.to(dev), ye.to(dev))
    table = {}
    clip = args.clip
    if clip <= 0.0:          # the median update norm of one warm-up round (clip norm too large to clip anything)
        torch.manual_seed(0)
        eng = FederatedEngine(resnet18(10), dev, backend="fused", lr=0.05, batch_size=128, logical_clients=n_clients,
                              sample_k=k, seed=5, dp_clip=1e30, dp_seed=17)
        eng.run_round(lambda c: shards[c], n_epoch=1, read_loss=False)
        norms = sorted(eng.last_update_norms())
        clip = norms[len(norms) // 2]
        print("utility clip = median update norm of a warm-up round = {:.4g}".format(clip), flush=True)
        del eng
        torch.cuda.empty_cache()
    for sigma in (0.0, 0.5, 1.0):
        torch.manual_seed(0)
        eng = FederatedEngine(resnet18(10), dev, backend="fused", lr=0.05, batch_size=128, logical_clients=n_clients,
                              sample_k=k, seed=5, dp_clip=clip, dp_noise_multiplier=sigma, dp_seed=17)
        for _ in range(args.utility_rounds):
            eng.run_round(lambda c: shards[c], n_epoch=1, read_loss=False)
        res = eng.evaluate(lambda c: held if c == 0 else None, batch_size=512)
        eps, order = eng.privacy_spent(1e-5)
        table[str(sigma)] = {"heldout_accuracy": round(res.accuracy, 4), "epsilon": eps, "order": order,
                             "mean_clip_factor": sum(eng.last_clip_factors()) / max(1, len(eng.last_clip_factors()))}
        print("utility sigma={} accuracy {:.4f} epsilon {:.3g}".format(sigma, res.accuracy, eps), flush=True)
        del eng
        torch.cuda.empty_cache()
    return {"clients": n_clients, "sampled": k, "client_samples": args.client_samples, "clip": clip,
            "rounds": args.utility_rounds, "delta": 1e-5, "by_sigma": table}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--rounds-per-rep", type=int, default=5)
    ap.add_argument("--utility-rounds", type=int, default=20)
    ap.add_argument("--client-samples", type=int, default=512)
    ap.add_argument("--clip", type=float, default=0.0, help="utility clip norm C (0: median update norm of a warm-up round)")
    ap.add_argument("--skip-utility", action="store_true")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("dp_bench.py measures on a CUDA device; none is available")
    dev = torch.device("cuda:0")
    out = card()
    out["cost"] = cost(args, torch, dev)
    if not args.skip_utility:
        out["utility"] = utility(args, torch, dev)
    out["sm_clock_after"] = card().get("sm_clock")
    print(json.dumps(out))


if __name__ == "__main__":
    main()
