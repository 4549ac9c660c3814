"""Robust aggregation (coordinate-wise median / trimmed mean, Multi-Krum) on the flagship configuration: what it costs
per round and what it does to accuracy under label-flipping and model-poisoning clients.

* round: ResNet-18, 1 GPU, one client, 4096 samples, batch 128, bf16 wire, 256 MiB L2 flush between rounds.  Engines with
  ``aggregator`` mean / median / trimmed_mean; blocks of device-timed rounds alternate between them (median + range).
* logical: 16 logical clients of 512 samples on one GPU, 8 sampled per round (the tile owner selects over 8 segments),
  mean against median and Multi-Krum (f = 2).
* collective: the robust and Krum kernels alone on ResNet-18's arena with P = 8, 16, 32 packed segments, against the
  plain one.
* utility: 16 Dirichlet(0.1) clients, 8 per round, 15 rounds, held-out accuracy for mean / median / trimmed_mean
  (beta = 0.25) / Multi-Krum (f = 2) with 0 attackers, 4 label-flipping attackers (their shards carry permuted labels)
  and 4 model-poisoning attackers (they upload -POISON_SCALE times their honest delta).  The poisoned rounds are driven
  here (train, rewrite theta, pack_client, aggregate) with every aggregator on a robust session; "mean" there is the
  trimmed mean with beta = 0, the unweighted mean, equal to the weighted one because every client holds as many samples.

    python scripts/robust_bench.py [--reps 5] [--rounds-per-rep 5] [--parts round,logical,collective] [--skip-utility]

Reads the card name, power limit and SM clock in the same run and prints one JSON line."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from fedprox_bench import card  # noqa: E402

AGGS = (("mean", {}), ("median", {"aggregator": "median"}),
        ("trimmed_mean", {"aggregator": "trimmed_mean", "trim_ratio": 0.25}))
KRUM = ("multi_krum", {"aggregator": "krum", "krum_f": 2})
POISON_SCALE = 4.0


def _alternate(torch, engines, run, reps, per_rep):
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda:0")

    def block(name, k):
        ms = []
        for _ in range(k):
            flush.zero_()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            run(engines[name])
            e1.record()
            e1.synchronize()
            ms.append(e0.elapsed_time(e1))
        return sorted(ms)[len(ms) // 2]
    names = list(engines)
    for name in names:
        block(name, 3)                                # capture + warm-up
    got = {name: [] for name in names}
    for r in range(reps):
        for name in (names if r % 2 == 0 else names[::-1]):
            got[name].append(block(name, per_rep))
    return {name: {"median_ms": sorted(v)[len(v) // 2], "range_ms": [min(v), max(v)]} for name, v in got.items()}


def round_cost(args, torch, dev):
    from baton_b200.data import dirichlet_label_shards, image_shard
    from baton_b200.models import resnet18
    from baton_b200.parallel.engine import FederatedEngine
    X, y = image_shard(dirichlet_label_shards(1, 10, 4096, alpha=0.5, seed=11)[0], seed=3, dtype=torch.bfloat16)
    shard = (X.to(dev), y.to(dev))
    engines = {}
    for name, kw in AGGS:
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


def logical_cost(args, torch, dev):
    from baton_b200.data import dirichlet_label_shards, image_shard
    from baton_b200.models import resnet18
    from baton_b200.parallel.engine import FederatedEngine
    specs = dirichlet_label_shards(16, 10, 512, alpha=0.5, seed=11)
    shards = {c: tuple(t.to(dev) for t in image_shard(specs[c], seed=3, dtype=torch.bfloat16)) for c in range(16)}
    engines = {}
    for name, kw in AGGS[:2] + (KRUM,):
        torch.manual_seed(0)
        engines[name] = FederatedEngine(resnet18(10), dev, backend="fused", lr=0.05, batch_size=128, n_ctas=132,
                                        seed=5, logical_clients=16, sample_k=8, **kw)

    def run(eng):
        eng.run_round(lambda c: shards[c], n_epoch=1, read_loss=False)
        eng.sync()
    out = _alternate(torch, engines, run, args.reps, 2)
    out["symmetric_bytes_median"] = 2 * engines["median"].session.half_wire
    del engines
    torch.cuda.empty_cache()
    return out


def collective_cost(args, torch, dev):
    from baton_b200.models import resnet18
    from baton_b200.parallel.arena import ParamArena
    from baton_b200.parallel.fedavg import FedAvgSession
    from baton_b200.parallel.robust import RobustConfig
    out = {}
    torch.manual_seed(0)
    arena = ParamArena(resnet18(10), dev, momentum=False)
    for label, cfg, P in [("mean", None, 1)] + [("median_P{}".format(p), RobustConfig("median"), p) for p in (8, 16, 32)] \
            + [("trimmed_P{}".format(p), RobustConfig("trimmed_mean", 0.25), p) for p in (8, 32)] \
            + [("krum_P{}".format(p), RobustConfig("krum", krum_f=2), p) for p in (8, 16, 32)]:
        sess = FedAvgSession(arena, wire_dtype="bf16", mode="delta", n_ctas=132, nvls=False, robust=cfg,
                             max_clients=P)
        ts = []
        for it in range(6):
            if cfg is not None:
                for j in range(P):
                    arena.theta.add_(1e-3)
                    sess.pack_client(j, reset=j + 1 < P)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            sess.aggregate(my_n=float(P), n_clients=P) if cfg is not None else sess.aggregate(my_n=1.0)
            e1.record()
            e1.synchronize()
            if it:
                ts.append(e0.elapsed_time(e1) * 1e3)
        sess.check()
        out[label] = {"median_us": sorted(ts)[len(ts) // 2], "range_us": [min(ts), max(ts)],
                      "read_bytes": P * sess._seg_bytes(arena.n)}
        del sess
        torch.cuda.empty_cache()
    return out


def utility(args, torch, dev):
    from baton_b200.data import dirichlet_label_shards, holdout_image_shard, image_shard
    from baton_b200.models import resnet18
    from baton_b200.parallel.engine import FederatedEngine
    n_clients, k = 16, 8
    specs = dirichlet_label_shards(n_clients, 10, args.client_samples, alpha=0.1, seed=11)
    clean = {c: tuple(t.to(dev) for t in image_shard(specs[c], seed=3, dtype=torch.bfloat16)) for c in range(n_clients)}
    Xe, ye = holdout_image_shard(10, 4096, seed=3, dtype=torch.bfloat16)
    held = (Xe.to(dev), ye.to(dev))
    perm = torch.tensor([3, 7, 0, 9, 5, 1, 8, 2, 6, 4], device=dev)       # the attackers' label map
    table = {}

    def poisoned_round(eng, n_bad):
        """One round with every participant packed by hand; attackers upload -POISON_SCALE x their honest delta."""
        a, sess = eng.arena, eng.session
        parts = eng.draw_participants()
        eng.sync()
        for j, cid in enumerate(parts):
            X, y = clean[cid]
            eng.trainer.run(X, y, n_epoch=1, return_device=True, **eng.hp)
            if cid < n_bad:
                a.theta.copy_(a.global_w - POISON_SCALE * (a.theta - a.global_w))
            sess.pack_client(j, reset=j + 1 < len(parts))
        sess.aggregate(my_n=float(len(parts)), n_clients=len(parts))

    for attack, n_bad in (("none", 0), ("label_flip", 4), ("model_poison", 4)):
        shards = {c: (clean[c][0], perm[clean[c][1]] if c < n_bad and attack == "label_flip" else clean[c][1])
                  for c in range(n_clients)}
        for name, kw in AGGS + (KRUM,):
            if attack == "model_poison" and name == "mean":
                kw = {"aggregator": "trimmed_mean", "trim_ratio": 0.0}
            torch.manual_seed(0)
            eng = FederatedEngine(resnet18(10), dev, backend="fused", lr=0.05, batch_size=128,
                                  logical_clients=n_clients, sample_k=k, seed=5, **kw)
            for _ in range(args.utility_rounds):
                if attack == "model_poison":
                    poisoned_round(eng, n_bad)
                else:
                    eng.run_round(lambda c: shards[c], n_epoch=1, read_loss=False)
            eng.session.check()
            res = eng.evaluate(lambda c: held if c == 0 else None, batch_size=512)
            table["{}{}_{}".format(attack, n_bad, name)] = round(res.accuracy, 4)
            print("utility attack={} attackers={} {:<12} accuracy {:.4f}".format(attack, n_bad, name, res.accuracy),
                  flush=True)
            del eng
            torch.cuda.empty_cache()
    return {"clients": n_clients, "sampled": k, "client_samples": args.client_samples, "alpha": 0.1,
            "rounds": args.utility_rounds, "trim_ratio": 0.25, "krum_f": 2, "poison_scale": POISON_SCALE,
            "heldout_accuracy": table}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--rounds-per-rep", type=int, default=5)
    ap.add_argument("--utility-rounds", type=int, default=15)
    ap.add_argument("--client-samples", type=int, default=512)
    ap.add_argument("--skip-utility", action="store_true")
    ap.add_argument("--parts", default="round,logical,collective", help="comma-separated cost parts to measure")
    args = ap.parse_args()
    parts = set(args.parts.split(","))
    import torch
    if not torch.cuda.is_available():
        sys.exit("robust_bench.py measures on a CUDA device; none is available")
    dev = torch.device("cuda:0")
    out = card()
    for name, fn in (("round", round_cost), ("logical", logical_cost), ("collective", collective_cost)):
        if name in parts:
            out[name] = fn(args, torch, dev)
            print(name, json.dumps(out[name]), flush=True)
    if not args.skip_utility:
        out["utility"] = utility(args, torch, dev)
    out["sm_clock_after"] = card().get("sm_clock")
    print(json.dumps(out))


if __name__ == "__main__":
    main()
