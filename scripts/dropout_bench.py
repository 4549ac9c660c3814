"""Dropout in BERT training: what the dropout forms of the kernels cost, and what dropout costs a round.

* kernels (CUDA events over 200 calls each, median of 5 blocks): the fused attention forward and backward at B=32,
  H=12, S=128 without and with dropout; the masked multi-kernel attention path (an all-zero attention mask) without
  and with dropout, forward and backward; the LayerNorm input-dropout and output-dropout pairs at [4096, 768] against
  the plain LayerNorm pair.
* rounds: a BERT-base round at bench.py's BERT configuration (1024 samples, batch 32, 5 local epochs, seq 128, SGD)
  with p = 0 and p = 0.1, in alternating blocks of device-timed rounds (the ``clip_bench.py`` method).

    python scripts/dropout_bench.py [--reps 5] [--rounds-per-rep 2] [--skip-rounds]

Reads the card name, power limit and SM clock in the same run and prints one JSON line."""
import argparse
import json
import math
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from fedprox_bench import card  # noqa: E402


def timed(torch, fn, calls=200, blocks=5):
    for _ in range(5):
        fn()
    per = []
    for _ in range(blocks):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(calls):
            fn()
        e1.record()
        e1.synchronize()
        per.append(e0.elapsed_time(e1) * 1e3 / calls)
    per.sort()
    return {"us": round(per[len(per) // 2], 2), "us_range": [round(per[0], 2), round(per[-1], 2)]}


def kernels(torch, dev):
    from baton_b200.data.dropout import DropoutRun
    from baton_b200.ops._ext import load
    C_ = load()
    run = DropoutRun()
    run.begin(0x1234, 7, 32, 5, 38)
    run.at(0, 3, torch.tensor([2, 7, 0], dtype=torch.int32, device=dev))
    da = run.kernel_args(1, 0.1)
    B, H, S, dh = 32, 12, 128, 64
    D = H * dh
    sc = 1.0 / math.sqrt(dh)
    g = torch.Generator(device=dev).manual_seed(0)
    qkv = torch.randn(B * S, 3 * D, device=dev, generator=g).to(torch.bfloat16)
    dout = torch.randn(B * S, D, device=dev, generator=g).to(torch.bfloat16)
    out = torch.empty(B * S, D, dtype=torch.bfloat16, device=dev)
    probs = torch.empty(B * H * S, S, dtype=torch.bfloat16, device=dev)
    dqkv = torch.empty_like(qkv)
    res = {}
    res["attn_fused_fwd"] = timed(torch, lambda: C_.attention_fwd(qkv, out, probs, B, S, H, dh, sc))
    res["attn_fused_fwd_drop"] = timed(torch, lambda: C_.attention_drop_fwd(qkv, out, probs, B, S, H, dh, sc, *da))
    res["attn_fused_bwd"] = timed(torch, lambda: C_.attention_bwd(qkv, dout, probs, dqkv, B, S, H, dh, sc))
    res["attn_fused_bwd_drop"] = timed(torch, lambda: C_.attention_drop_bwd(qkv, dout, probs, dqkv, B, S, H, dh, sc, *da))
    # the masked multi-kernel path through the autograd function (an all-zero additive mask)
    from baton_b200.ops.nn import _AttnFn
    mask = torch.zeros(B, S, device=dev)
    x = qkv.clone().requires_grad_(True)

    def multi(dargs):
        def f():
            o = _AttnFn.apply(x, B, S, H, dh, mask, dargs)
            o.backward(dout)
        return f
    res["attn_multi_fwd_bwd"] = timed(torch, multi(None), calls=50)
    res["attn_multi_fwd_bwd_drop"] = timed(torch, multi(da), calls=50)
    rows, C = 4096, 768
    xs = torch.randn(rows, C, device=dev, generator=g).to(torch.bfloat16)
    rs = torch.randn(rows, C, device=dev, generator=g).to(torch.bfloat16)
    dy = torch.randn(rows, C, device=dev, generator=g).to(torch.bfloat16)
    gam, bet = torch.randn(C, device=dev), torch.randn(C, device=dev)
    y, pre, dx, dxd = (torch.empty_like(xs) for _ in range(4))
    mean, rstd = torch.empty(rows, device=dev), torch.empty(rows, device=dev)
    dg, db = torch.zeros(C, device=dev), torch.zeros(C, device=dev)

    def ln_in():
        C_.layernorm_drop_fwd(xs, rs, y, pre, gam, bet, mean, rstd, rows, C, 1e-12, 1, *da)
        C_.layernorm_drop_bwd(pre, dy, dx, dxd, gam, mean, rstd, dg, db, rows, C, 1, *da)

    def ln_out():
        C_.layernorm_drop_fwd(xs, rs, y, None, gam, bet, mean, rstd, rows, C, 1e-12, 2, *da)
        C_.layernorm_drop_bwd(pre, dy, dx, None, gam, mean, rstd, dg, db, rows, C, 2, *da)
    from baton_b200.ops import functional as F

    def ln_plain_pair():
        C_.layernorm_fwd(xs, rs, y, gam, bet, mean, rstd, rows, C, 1e-12)
        F.add(xs, rs)
        C_.layernorm_bwd(pre, dy, dx, gam, mean, rstd, dg, db, rows, C)
    res["ln_pair_plain_with_add"] = timed(torch, ln_plain_pair)
    res["ln_pair_input_dropout"] = timed(torch, ln_in)
    res["ln_pair_output_dropout"] = timed(torch, ln_out)
    return res


def rounds(torch, dev, args):
    from baton_b200.data import dirichlet_label_shards, token_shard
    from baton_b200.models import bert_base
    from baton_b200.parallel.engine import FederatedEngine
    engines = {}
    for k, p in (("p0", 0.0), ("p0.1", 0.1)):
        torch.manual_seed(0)
        engines[k] = FederatedEngine(bert_base(2, hidden_dropout_prob=p, attention_probs_dropout_prob=p), dev,
                                     backend="fused", lr=2e-5, batch_size=32, n_ctas=132, seed=5)
    spec = dirichlet_label_shards(1, 2, 1024, alpha=0.5, seed=11)[0]
    X, y = token_shard(spec, seq_len=128, vocab=engines["p0"].model.config.vocab_size, seed=3)
    shard = (X.to(dev), y.to(dev))
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)

    def block(k, m):
        ms = []
        for _ in range(m):
            flush.zero_()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            engines[k].run_round(shard, n_epoch=5, read_loss=False)
            engines[k].sync()
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
            print("rep {} {:<5} {:.3f} ms/round".format(r, k, reps[k][-1]), flush=True)
    out = {}
    for k, v in reps.items():
        out["round_ms_" + k] = round(sorted(v)[len(v) // 2], 2)
        out["round_ms_range_" + k] = [round(min(v), 2), round(max(v), 2)]
    out["overhead"] = round(out["round_ms_p0.1"] / out["round_ms_p0"] - 1.0, 4)
    out["kernels_per_epoch"] = {k: e.trainer.kernels_per_epoch for k, e in engines.items()}
    out["config"] = "bert_base, 1024 samples, batch 32, 5 local epochs, seq 128, sgd lr 2e-5"
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--rounds-per-rep", type=int, default=2)
    ap.add_argument("--skip-rounds", action="store_true")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("dropout_bench.py measures on a CUDA device; none is available")
    dev = torch.device("cuda:0")
    out = card()
    out["kernels"] = kernels(torch, dev)
    print(json.dumps(out["kernels"]), flush=True)
    if not args.skip_rounds:
        torch.cuda.empty_cache()
        out["rounds_bert_base"] = rounds(torch, dev, args)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
