"""Gradient-norm clipping: what the norm kernel costs, and what clipping costs a round.

* norm kernel alone (``F.grad_norm_clip``): CUDA events over 200 launches on the ResNet-18 arena (11.18 M parameters,
  44.7 MB read per launch) and the BERT-base arena (about 438 MB), after a 256 MiB L2 flush per launch-block;
  the achieved read bandwidth is the bytes over the kernel time.
* rounds: device-timed rounds, clipping off and on (at a threshold that clips most steps) in alternating blocks, the
  ``adamw_bench.py`` method:
  - ResNet-18 flagship: 1 GPU, 4096 samples, batch 128 (32 steps), 1 local epoch, SGD lr 0.05;
  - BERT-base at bench.py's BERT configuration (1024 samples, batch 32, 5 local epochs, seq 128) with AdamW.

    python scripts/clip_bench.py [--reps 5] [--rounds-per-rep 3] [--skip-bert]

Reads the card name, power limit and SM clock in the same run and prints one JSON line."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from fedprox_bench import card  # noqa: E402


def norm_kernel(torch, dev, n, launches=200):
    from baton_b200.ops import functional as F
    g = torch.randn(n, device=dev) * 1e-3
    work = torch.zeros(F.load().GRAD_NORM_WORK_WORDS, dtype=torch.int64, device=dev)
    c = torch.tensor([1.0], device=dev)
    out = torch.zeros(2, device=dev)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    for _ in range(10):
        F.grad_norm_clip(g, c, work, out[0:1], out[1:2])
    per = []
    for _ in range(5):
        flush.zero_()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(launches):
            F.grad_norm_clip(g, c, work, out[0:1], out[1:2])
        e1.record()
        e1.synchronize()
        per.append(e0.elapsed_time(e1) * 1e3 / launches)
    us = sorted(per)[len(per) // 2]
    return {"n_param": n, "bytes": 4 * n, "us": round(us, 2), "us_range": [round(min(per), 2), round(max(per), 2)],
            "read_GBps": round(4 * n / us / 1e3, 1)}


def rounds(torch, engines, shard, n_epoch, args):
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=shard[0].device)

    def block(k, m):
        eng = engines[k]
        ms = []
        for _ in range(m):
            flush.zero_()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            eng.run_round(shard, n_epoch=n_epoch, read_loss=False)
            eng.sync()
            e1.record()
            e1.synchronize()
            ms.append(e0.elapsed_time(e1))
        return sorted(ms)[len(ms) // 2]

    keys = list(engines)
    for k in keys:
        block(k, 2)                                   # capture + warm-up
    reps = {k: [] for k in keys}
    for r in range(args.reps):
        for k in (keys if r % 2 == 0 else keys[::-1]):
            reps[k].append(block(k, args.rounds_per_rep))
            print("rep {} {:<4} {:.3f} ms/round".format(r, k, reps[k][-1]), flush=True)
    out = {}
    for k, v in reps.items():
        out["round_ms_" + k] = sorted(v)[len(v) // 2]
        out["round_ms_range_" + k] = [min(v), max(v)]
    out["overhead"] = out["round_ms_clip"] / out["round_ms_off"] - 1.0
    norms = [x for r in engines["clip"].last_grad_norms()[0] for x in r]
    out["clip_threshold"] = engines["clip"].hp["max_grad_norm"]
    out["steps_clipped"] = "{}/{}".format(sum(x > out["clip_threshold"] for x in norms), len(norms))
    out["grad_norm_range"] = [min(norms), max(norms)]
    return out


def resnet(args, torch, dev):
    from baton_b200.data import dirichlet_label_shards, image_shard
    from baton_b200.models import resnet18
    from baton_b200.parallel.engine import FederatedEngine
    spec = dirichlet_label_shards(1, 10, 4096, alpha=0.5, seed=11)[0]
    X, y = image_shard(spec, seed=3, dtype=torch.bfloat16)
    engines = {}
    for k, C in (("off", 0.0), ("clip", args.resnet_clip)):
        torch.manual_seed(0)
        engines[k] = FederatedEngine(resnet18(10), dev, backend="fused", lr=0.05, batch_size=128, n_ctas=132, seed=5,
                                     max_grad_norm=C)
    out = rounds(torch, engines, (X.to(dev), y.to(dev)), 1, args)
    out["config"] = "resnet18, 4096 samples, batch 128 (32 steps), 1 local epoch, sgd lr 0.05"
    return out


def bert(args, torch, dev):
    from baton_b200.data import dirichlet_label_shards, token_shard
    from baton_b200.models import bert_base
    from baton_b200.parallel.engine import FederatedEngine
    engines = {}
    for k, C in (("off", 0.0), ("clip", args.bert_clip)):
        torch.manual_seed(0)
        engines[k] = FederatedEngine(bert_base(2), dev, backend="fused", lr=2e-5, batch_size=32, n_ctas=132, seed=5,
                                     optimizer="adamw", max_grad_norm=C)
    spec = dirichlet_label_shards(1, 2, 1024, alpha=0.5, seed=11)[0]
    X, y = token_shard(spec, seq_len=128, vocab=engines["off"].model.config.vocab_size, seed=3)
    out = rounds(torch, engines, (X.to(dev), y.to(dev)), 5, args)
    out["config"] = "bert_base, 1024 samples, batch 32, 5 local epochs, seq 128, adamw lr 2e-5"
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--rounds-per-rep", type=int, default=3)
    ap.add_argument("--resnet-clip", type=float, default=0.05)
    ap.add_argument("--bert-clip", type=float, default=1e-8)     # this configuration's gradient norms are ~1e-7
    ap.add_argument("--skip-bert", action="store_true")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("clip_bench.py measures on a CUDA device; none is available")
    dev = torch.device("cuda:0")
    out = card()
    from baton_b200.models import bert_base, resnet18
    from baton_b200.parallel.arena import ParamArena
    for name, mk in (("resnet18", lambda: resnet18(10)), ("bert_base", lambda: bert_base(2))):
        n = ParamArena(mk(), torch.device("cpu")).n_param
        out["norm_kernel_" + name] = norm_kernel(torch, dev, n)
        print(name, out["norm_kernel_" + name], flush=True)
    out["rounds_resnet18"] = resnet(args, torch, dev)
    torch.cuda.empty_cache()
    if not args.skip_bert:
        out["rounds_bert_base"] = bert(args, torch, dev)
    out["sm_clock_after"] = card().get("sm_clock")
    print(json.dumps(out))


if __name__ == "__main__":
    main()
