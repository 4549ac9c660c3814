"""What random-crop / flip augmentation costs: the augmenting gather kernel against the plain one, and a flagship round
with augmentation off against on.

* kernel: ``F.gather_rows`` and ``F.gather_augment`` (``crop_flip``, padding 4) on the flagship epoch shard, 4096
  samples of 32x32x3 bf16 gathered through a random permutation.  CUDA events around blocks of ``--launches``
  back-to-back launches, the two kernels in alternating blocks; per kernel the median time per launch and the
  achieved bytes/s (the shard read once plus the output written once) against the H100 SXM's 3.35 TB/s.
* round: bench.py's default config (ResNet-18, 1 GPU, 4096 samples, batch 128, one local epoch, fused backend),
  engines with ``augment=None`` and ``augment="crop_flip"`` in alternating blocks, device-timed rounds with a 256 MiB
  L2 flush before each; per setting the median round time and the range over the blocks.

    python scripts/augment_bench.py [--launches 200] [--kernel-reps 10] [--reps 5] [--rounds-per-rep 3]

Reads the card name, power limit and SM clock in the same run and prints one JSON line."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from fedprox_bench import card  # noqa: E402

HBM_BPS = 3.35e12          # H100 SXM data sheet


def kernel(args, torch, dev):
    from baton_b200.data.augment import augment_key, epoch_words
    from baton_b200.ops import functional as F
    n = 4096
    X = torch.randn(n, 32, 32, 3, device=dev).to(torch.bfloat16)
    perm = torch.randperm(n, device=dev)
    out = torch.empty_like(X)
    words = epoch_words(1, 1).to(dev)[0]
    key = augment_key(0)
    run = {"gather_rows": lambda: F.gather_rows(X, perm, out=out),
           "gather_augment": lambda: F.gather_augment(X, perm, words, key, 4, crop=True, flip=True, out=out)}

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
    for r in range(args.kernel_reps):
        for name in (list(run) if r % 2 == 0 else list(run)[::-1]):
            us[name].append(block(name))
    moved = 2 * X.numel() * X.element_size()                 # read + write of the kept bytes
    res = {"shard": "4096 x 32x32x3 bf16", "bytes_moved": moved, "launches_per_block": args.launches}
    for name, v in us.items():
        med = sorted(v)[len(v) // 2]
        res[name] = {"us_median": round(med, 2), "us_range": [round(min(v), 2), round(max(v), 2)],
                     "TBps": round(moved / med / 1e6, 3), "share_of_3.35TBps": round(moved / med / 1e-6 / HBM_BPS, 3)}
    res["augment_over_rows"] = round(res["gather_augment"]["us_median"] / res["gather_rows"]["us_median"], 3)
    return res


def rounds(args, torch, dev):
    from baton_b200.data import ShardSpec, image_shard
    from baton_b200.models import resnet18
    from baton_b200.parallel.engine import FederatedEngine
    X, y = image_shard(ShardSpec(0, torch.full((10,), 0.1), 4096), seed=3, dtype=torch.bfloat16)
    shard = (X.to(dev), y.to(dev))
    engines = {}
    for aug in ("none", "crop_flip"):
        torch.manual_seed(0)
        engines[aug] = FederatedEngine(resnet18(10), dev, backend="fused", lr=0.05, batch_size=128, n_ctas=132,
                                       seed=5, augment=None if aug == "none" else aug)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)

    def block(aug, k):
        eng = engines[aug]
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

    for aug in engines:
        block(aug, 2)                                        # capture + warm-up
    reps = {aug: [] for aug in engines}
    for r in range(args.reps):
        for aug in (list(engines) if r % 2 == 0 else list(engines)[::-1]):
            reps[aug].append(block(aug, args.rounds_per_rep))
            print("round rep {} {:<9} {:.3f} ms".format(r, aug, reps[aug][-1]), flush=True)
    out = {"config": "resnet18, 4096 samples, batch 128, 1 local epoch, fused, 1 GPU"}
    for aug, v in reps.items():
        out["round_ms_" + aug] = round(sorted(v)[len(v) // 2], 3)
        out["round_ms_range_" + aug] = [round(min(v), 3), round(max(v), 3)]
    out["overhead"] = round(out["round_ms_crop_flip"] / out["round_ms_none"] - 1.0, 4)
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
        sys.exit("augment_bench.py measures on a CUDA device; none is available")
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
