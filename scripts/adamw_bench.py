"""Local AdamW against local SGD: what AdamW costs per round, and what it does on a BERT task.

* cost: device-timed rounds, SGD and AdamW engines in alternating blocks (both epoch graphs are captured during
  warm-up), 256 MiB L2 flush between rounds as bench.py does; per setting the median round time and the range over
  the blocks.  Two configurations:
  - ResNet-18 flagship: 1 GPU, 4096 samples, batch 128, 1 local epoch, bf16, resident shard;
  - BERT-base at bench.py's BERT config: 1024 samples, batch 32, 5 local epochs, sequence length 128.
* utility: bert_tiny, 4 clients on one GPU (logical clients), 256 token samples each (Dirichlet alpha = 0.5), the
  same seeds for SGD and AdamW at their own learning rates; held-out accuracy on ``holdout_token_shard`` after
  every round.

    python scripts/adamw_bench.py [--reps 5] [--rounds-per-rep 3] [--effect-rounds 6] [--skip-bert-cost]

Reads the card name, power limit and SM clock in the same run and prints one JSON line."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from fedprox_bench import card  # noqa: E402

OPTS = ("sgd", "adamw")


def _timed_blocks(torch, engines, shard, n_epoch, args):
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=shard[0].device)

    def block(opt, k):
        eng = engines[opt]
        ms = []
        for _ in range(k):
            flush.zero_()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            eng.run_round(shard, n_epoch=n_epoch, read_loss=False)
            eng.sync()
            e1.record()
            e1.synchronize()
            ms.append(e0.elapsed_time(e1))
        return sorted(ms)[len(ms) // 2]

    for opt in OPTS:
        block(opt, 2)                                 # capture + warm-up
    reps = {opt: [] for opt in OPTS}
    for r in range(args.reps):
        for opt in (OPTS if r % 2 == 0 else OPTS[::-1]):
            reps[opt].append(block(opt, args.rounds_per_rep))
            print("cost rep {} {:<5} {:.3f} ms/round".format(r, opt, reps[opt][-1]), flush=True)
    out = {}
    for opt, v in reps.items():
        out["round_ms_" + opt] = sorted(v)[len(v) // 2]
        out["round_ms_range_" + opt] = [min(v), max(v)]
    out["overhead"] = out["round_ms_adamw"] / out["round_ms_sgd"] - 1.0
    return out


def cost_resnet(args, torch, dev):
    from baton_b200.data import dirichlet_label_shards, image_shard
    from baton_b200.models import resnet18
    from baton_b200.parallel.engine import FederatedEngine
    spec = dirichlet_label_shards(1, 10, 4096, alpha=0.5, seed=11)[0]
    X, y = image_shard(spec, seed=3, dtype=torch.bfloat16)
    shard = (X.to(dev), y.to(dev))
    engines = {}
    for opt, lr in (("sgd", 0.05), ("adamw", 1e-3)):
        torch.manual_seed(0)
        engines[opt] = FederatedEngine(resnet18(10), dev, backend="fused", lr=lr, batch_size=128, n_ctas=132, seed=5,
                                       optimizer=opt)
    out = _timed_blocks(torch, engines, shard, 1, args)
    out["config"] = "resnet18, 4096 samples, batch 128, 1 local epoch"
    return out


def cost_bert(args, torch, dev):
    from baton_b200.data import dirichlet_label_shards, token_shard
    from baton_b200.models import bert_base
    from baton_b200.parallel.engine import FederatedEngine
    engines = {}
    for opt, lr in (("sgd", 0.05), ("adamw", 2e-5)):
        torch.manual_seed(0)
        engines[opt] = FederatedEngine(bert_base(2), dev, backend="fused", lr=lr, batch_size=32, n_ctas=132, seed=5,
                                       optimizer=opt)
    spec = dirichlet_label_shards(1, 2, 1024, alpha=0.5, seed=11)[0]
    X, y = token_shard(spec, seq_len=128, vocab=engines["sgd"].model.config.vocab_size, seed=3)
    out = _timed_blocks(torch, engines, (X.to(dev), y.to(dev)), 5, args)
    out["config"] = "bert_base, 1024 samples, batch 32, 5 local epochs, seq 128"
    out["adamw_state_bytes"] = engines["adamw"].arena.adam_v.numel() * 4
    return out


def effect(args, torch, dev):
    from baton_b200.data import dirichlet_label_shards, holdout_token_shard, token_shard
    from baton_b200.models import bert_tiny
    from baton_b200.parallel.engine import FederatedEngine
    n_clients, classes = 4, 2
    specs = dirichlet_label_shards(n_clients, classes, 256, alpha=0.5, seed=11)
    vocab = bert_tiny(classes).config.vocab_size
    shards = {c: tuple(t.to(dev) for t in token_shard(specs[c], seq_len=64, vocab=vocab, seed=3))
              for c in range(n_clients)}
    Xe, ye = holdout_token_shard(classes, 1024, seq_len=64, vocab=vocab, seed=3)
    held = (Xe.to(dev), ye.to(dev))
    curves, lrs = {}, {"sgd": args.sgd_lr, "adamw": args.adamw_lr}
    for opt in OPTS:
        torch.manual_seed(0)
        eng = FederatedEngine(bert_tiny(classes), dev, backend="fused", lr=lrs[opt], batch_size=32,
                              logical_clients=n_clients, seed=5, optimizer=opt, weight_decay=0.01 if opt == "adamw" else 0)
        acc = []
        for rnd in range(1, args.effect_rounds + 1):
            eng.run_round(lambda c: shards[c], n_epoch=2, read_loss=False)
            res = eng.evaluate(lambda c: held if c == 0 else None, batch_size=256)
            acc.append(round(res.accuracy, 4))
            print("effect {:<5} round {:2d} held-out accuracy {:.4f}".format(opt, rnd, res.accuracy), flush=True)
        curves[opt] = acc
        del eng
        torch.cuda.empty_cache()
    return {"model": "bert_tiny", "clients": n_clients, "client_samples": 256, "alpha": 0.5, "seq_len": 64,
            "local_epochs": 2, "batch": 32, "lr": lrs, "adamw_weight_decay": 0.01, "heldout_accuracy": curves}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--rounds-per-rep", type=int, default=3)
    ap.add_argument("--effect-rounds", type=int, default=6)
    ap.add_argument("--sgd-lr", type=float, default=0.05)
    ap.add_argument("--adamw-lr", type=float, default=1e-3)
    ap.add_argument("--skip-bert-cost", action="store_true")
    ap.add_argument("--skip-effect", action="store_true")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("adamw_bench.py measures on a CUDA device; none is available")
    dev = torch.device("cuda:0")
    out = card()
    out["cost_resnet18"] = cost_resnet(args, torch, dev)
    torch.cuda.empty_cache()
    if not args.skip_bert_cost:
        out["cost_bert_base"] = cost_bert(args, torch, dev)
        torch.cuda.empty_cache()
    if not args.skip_effect:
        out["effect"] = effect(args, torch, dev)
    out["sm_clock_after"] = card().get("sm_clock")
    print(json.dumps(out))


if __name__ == "__main__":
    main()
