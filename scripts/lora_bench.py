"""LoRA costs on one GPU: the adapter kernels against the plain GEMM at BERT-base shapes, and a BERT-base round at
bench.py's BERT configuration (1024 samples, batch 32, 5 local epochs, sequence 128, AdamW) with full fine-tuning
against LoRA r = 8 on query / value, in alternating blocks.  Prints one JSON line and writes it to --out, with the card
name and power limit the numbers were measured at.

    python scripts/lora_bench.py --out /tmp/lora_bench.json
"""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       stdout=subprocess.PIPE, text=True).stdout.strip().splitlines()
    return q[0] if q else "unknown"


def time_us(fn, iters=50, warmup=10):
    for _ in range(warmup):
        fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1e3 / iters


def kernels(dev):
    from baton_b200.ops import functional as F
    out = {}
    M, R, r = 4096, 16, 8
    for K, N, name in ((768, 2304, "qkv K=768 N=2304 (q,v)"), (3072, 768, "ffn_out K=3072 N=768")):
        x = torch.randn(M, K, device=dev).to(torch.bfloat16)
        w = (torch.randn(N, K, device=dev) * 0.02).to(torch.bfloat16)
        a = (torch.randn(R, K, device=dev) * 0.02).to(torch.bfloat16)
        ds = N // 3 if N == 2304 else N
        slot = (0, -1, 1) if N == 2304 else (0, -1, -1)
        rs = r if N == 2304 else R
        bb = (torch.randn((2 if N == 2304 else 1) * ds, rs, device=dev) * 0.02).to(torch.bfloat16)
        u = F.lora_down(x, a, T=1, rs=R, kt=K, xoff=(0,), w_ts=0, wsj=K, wsk=1)
        dy = torch.randn(M, N, device=dev).to(torch.bfloat16)
        lo = [0, 2 * ds] if N == 2304 else [0]
        T = len(lo)
        v = F.lora_down(dy, bb, T=T, rs=rs, kt=ds, xoff=lo, w_ts=ds * rs, wsj=1, wsk=rs)
        ga = torch.zeros(R, K, device=dev)
        gb = torch.zeros(T * ds, rs, device=dev)
        lora_f = dict(u=u, f=bb, fs_n=rs, fs_j=1, rs=rs, ds=ds, slot=slot, s=2.0)
        lora_d = dict(u=v, f=a, fs_n=1, fs_j=K, rs=R, ds=K, slot=(0, -1, -1), s=2.0)
        out[name] = {
            "gemm_fwd_us": time_us(lambda: F.gemm(x, w)),
            "gemm_lora_fwd_us": time_us(lambda: F.gemm_lora(x, w, lora_f)),
            "gemm_dgrad_us": time_us(lambda: F.gemm(dy, w, b_mn=True)),
            "gemm_lora_dgrad_us": time_us(lambda: F.gemm_lora(dy, w, lora_d, b_mn=True)),
            "wgrad_us": time_us(lambda: F.gemm(dy, x, a_mn=True, b_mn=True, out=torch.empty(N, K, device=dev),
                                               accumulate=True)),
            "lora_down_U_us": time_us(lambda: F.lora_down(x, a, T=1, rs=R, kt=K, xoff=(0,), w_ts=0, wsj=K, wsk=1)),
            "lora_down_V_us": time_us(lambda: F.lora_down(dy, bb, T=T, rs=rs, kt=ds, xoff=lo, w_ts=ds * rs, wsj=1,
                                                          wsk=rs)),
            "lora_dA_us": time_us(lambda: F.lora_grad_(x, v, ga, NA=K, NB=R, lo=(0,), qo=(0,), osa=1, osb=K, out_ts=0,
                                                       s=2.0)),
            "lora_dB_us": time_us(lambda: F.lora_grad_(dy, u, gb, NA=ds, NB=rs, lo=lo, qo=[t * rs for t in range(T)],
                                                       osa=rs, osb=1, out_ts=ds * rs, s=2.0)),
        }
    return out


def rounds(dev, blocks, rounds_per_block):
    from baton_b200.models.bert import LoraConfig, bert_base
    from baton_b200.parallel.engine import FederatedEngine
    g = torch.Generator().manual_seed(0)
    X = torch.randint(0, 30522, (1024, 128), generator=g).to(dev)
    y = (X[:, :4].sum(1) % 2).to(dev)
    engines = {}
    for name, lora in (("full", None), ("lora_r8_qv", LoraConfig(8, 16))):
        torch.manual_seed(0)
        engines[name] = FederatedEngine(bert_base(2, lora=lora), dev, backend="fused", lr=1e-4, batch_size=32,
                                        optimizer="adamw")
    times = {k: [] for k in engines}
    for e in engines.values():        # warm-up: graph capture and first launches
        e.run_round((X, y), n_epoch=5)
        e.sync()
    for _ in range(blocks):
        for name, e in engines.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in range(rounds_per_block):
                e.run_round((X, y), n_epoch=5)
            e.sync()
            torch.cuda.synchronize()
            times[name].append((time.perf_counter() - t0) / rounds_per_block)
    out = {}
    for name, e in engines.items():
        t = sorted(times[name])
        out[name] = {"round_s_median": t[len(t) // 2], "round_s_min": t[0], "round_s_max": t[-1],
                     "wire_bytes": e.last_upload_bytes(),
                     "kernels_per_epoch": getattr(e.trainer, "kernels_per_epoch", None),
                     "trainable_params": sum(p.numel() for p in e.model.parameters() if p.requires_grad)}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--blocks", type=int, default=3)
    ap.add_argument("--rounds-per-block", type=int, default=1)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("lora_bench needs a GPU")
    dev = torch.device("cuda:0")
    res = {"card": card(), "kernels": kernels(dev), "bert_base_round": rounds(dev, args.blocks, args.rounds_per_block)}
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
