"""What mixup / CutMix / label smoothing cost: the mixing gather kernel against the augmenting one, and a flagship round
with each option against none.

* kernel: ``F.gather_augment`` (``crop_flip``, padding 4) plainly and with mixup / CutMix rows (``mix_rows``, batch
  128) on the flagship epoch shard, 4096 samples of 32x32x3 bf16 gathered through a random permutation.  CUDA events
  around blocks of ``--launches`` back-to-back launches, the kernels in alternating blocks; per kernel the median time
  per launch.  The mixing gather reads two images per output (its own and its partner's).
* round: bench.py's default config (ResNet-18, 1 GPU, 4096 samples, batch 128, one local epoch, fused backend),
  engines with ``mix=None``, ``"mixup"``, ``"cutmix"`` and ``label_smoothing=0.1`` in alternating blocks, device-timed
  rounds with a 256 MiB L2 flush before each; per setting the median round time and the range over the blocks.

    python scripts/mix_bench.py [--launches 200] [--kernel-reps 10] [--reps 5] [--rounds-per-rep 3]

Reads the card name, power limit and SM clock in the same run and prints one JSON line."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from fedprox_bench import card  # noqa: E402

ROUND_SETTINGS = {"none": {}, "mixup": dict(mix="mixup"), "cutmix": dict(mix="cutmix"),
                  "smoothing": dict(label_smoothing=0.1)}


def kernel(args, torch, dev):
    from baton_b200.data.augment import augment_key, epoch_words
    from baton_b200.data.mix import MixConfig, mix_table
    from baton_b200.ops import functional as F
    n, bs = 4096, 128
    X = torch.randn(n, 32, 32, 3, device=dev).to(torch.bfloat16)
    perm = torch.randperm(n, device=dev)
    out = torch.empty_like(X)
    words = epoch_words(1, 1).to(dev)[0]
    key = augment_key(0)
    rows = {k: torch.from_numpy(mix_table(key, 1, 0, n // bs, MixConfig(k, 1.0, 0.0), 32, 32)).to(dev)
            for k in ("mixup", "cutmix")}
    run = {"gather_augment": lambda: F.gather_augment(X, perm, words, key, 4, out=out),
           "gather_mix_mixup": lambda: F.gather_augment(X, perm, words, key, 4, out=out, mix_rows=rows["mixup"],
                                                        batch=bs),
           "gather_mix_cutmix": lambda: F.gather_augment(X, perm, words, key, 4, out=out, mix_rows=rows["cutmix"],
                                                         batch=bs)}

    def block(name):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(args.launches):
            run[name]()
        e1.record()
        e1.synchronize()
        return e0.elapsed_time(e1) * 1e3 / args.launches     # us per launch

    for name in run:
        block(name)                                          # warm-up
    us = {name: [] for name in run}
    names = list(run)
    for r in range(args.kernel_reps):
        for name in (names if r % 2 == 0 else names[::-1]):
            us[name].append(block(name))
    res = {"shard": "4096 x 32x32x3 bf16, batch 128, crop_flip padding 4", "launches_per_block": args.launches}
    for name, v in us.items():
        res[name] = {"us_median": round(sorted(v)[len(v) // 2], 2), "us_range": [round(min(v), 2), round(max(v), 2)]}
    for name in names[1:]:
        res[name + "_over_augment"] = round(res[name]["us_median"] / res["gather_augment"]["us_median"], 3)
    return res


def rounds(args, torch, dev):
    from baton_b200.data import ShardSpec, image_shard
    from baton_b200.models import resnet18
    from baton_b200.parallel.engine import FederatedEngine
    X, y = image_shard(ShardSpec(0, torch.full((10,), 0.1), 4096), seed=3, dtype=torch.bfloat16)
    shard = (X.to(dev), y.to(dev))
    engines = {}
    for name, kw in ROUND_SETTINGS.items():
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
        block(name, 2)                                       # capture + warm-up
    reps = {name: [] for name in engines}
    names = list(engines)
    for r in range(args.reps):
        for name in (names if r % 2 == 0 else names[::-1]):
            reps[name].append(block(name, args.rounds_per_rep))
            print("round rep {} {:<9} {:.3f} ms".format(r, name, reps[name][-1]), flush=True)
    out = {"config": "resnet18, 4096 samples, batch 128, 1 local epoch, fused, 1 GPU"}
    for name, v in reps.items():
        out["round_ms_" + name] = round(sorted(v)[len(v) // 2], 3)
        out["round_ms_range_" + name] = [round(min(v), 3), round(max(v), 3)]
    for name in names[1:]:
        out["overhead_" + name] = round(out["round_ms_" + name] / out["round_ms_none"] - 1.0, 4)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=200)
    ap.add_argument("--kernel-reps", type=int, default=10)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--rounds-per-rep", type=int, default=3)
    ap.add_argument("--out", default=None, help="also write the JSON result to this file")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("mix_bench.py measures on a CUDA device; none is available")
    dev = torch.device("cuda:0")
    out = card()
    out["kernel"] = kernel(args, torch, dev)
    print("kernel: {}".format(json.dumps(out["kernel"])), flush=True)
    out["round"] = rounds(args, torch, dev)
    line = json.dumps(out)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
