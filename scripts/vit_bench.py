"""Vision Transformer kernels and rounds on one GPU, with CUDA events, in alternating blocks after a warm-up.

    python scripts/vit_bench.py [--reps 5] [--iters 50] [--rounds 3]

1. The short-S fused attention (S = 65, d_head = 64, B = 128, H = 3 and 6), forward and forward + backward, against
   ``torch.nn.functional.scaled_dot_product_attention`` on the same bf16 shapes (``[B, H, S, 64]`` views).
2. The add + LayerNorm pair (forward + backward) and the token kernel (forward + backward) at ``[128*65, 192]`` and
   ``[128*65, 384]``.
3. One federated round on one GPU (4096 Dirichlet(0.5) samples, batch 128, one local epoch, captured epoch graph) for
   vit_tiny and resnet18, alternating.
Prints the card name and power limit, then one JSON line per measurement (median over blocks, milliseconds)."""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

BF16 = torch.bfloat16
DEV = torch.device("cuda:0")


def card():
    name = torch.cuda.get_device_name(DEV)
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                            stdout=subprocess.PIPE, text=True, timeout=30).stdout.strip()
    except Exception as exc:        # the number stays unlabelled rather than guessed
        pl = "unknown ({})".format(exc)
    return name, pl


def timed(fn, iters):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(iters):
        fn()
    e.record()
    e.synchronize()
    return s.elapsed_time(e) / iters


def alternate(cases, reps, iters):
    """{name: median ms per call} over ``reps`` blocks, the cases taking turns inside each block"""
    for fn in cases.values():
        fn()
    torch.cuda.synchronize()
    out = {k: [] for k in cases}
    for _ in range(reps):
        for k, fn in cases.items():
            out[k].append(timed(fn, iters))
    return {k: statistics.median(v) for k, v in out.items()}


def emit(**kw):
    print(json.dumps(kw), flush=True)


def attention(args):
    from baton_b200.ops import load
    C = load()
    B, S = 128, 65
    for H in (3, 6):
        D = H * 64
        torch.manual_seed(0)
        qkv = torch.randn(B * S, 3 * D, device=DEV).to(BF16)
        dout = torch.randn(B * S, D, device=DEV).to(BF16)
        out = torch.empty(B * S, D, device=DEV, dtype=BF16)
        probs = torch.empty(B * H, S, (S + 7) // 8 * 8, device=DEV, dtype=BF16)
        dqkv = torch.empty_like(qkv)
        q, k, v = (t.reshape(B, S, H, 64).transpose(1, 2).detach().requires_grad_() for t in qkv.split(D, dim=-1))
        g = dout.reshape(B, S, H, 64).transpose(1, 2)
        F = torch.nn.functional

        def ours_f():
            C.attention_short_fwd(qkv, out, probs, B, S, H, 64, 0.125)

        def ours_fb():
            C.attention_short_fwd(qkv, out, probs, B, S, H, 64, 0.125)
            C.attention_short_bwd(qkv, dout, probs, dqkv, B, S, H, 64, 0.125)

        def sdpa_f():
            with torch.no_grad():
                F.scaled_dot_product_attention(q, k, v)

        def sdpa_fb():
            o = F.scaled_dot_product_attention(q, k, v)
            torch.autograd.grad(o, (q, k, v), g)

        r = alternate({"ours_fwd": ours_f, "sdpa_fwd": sdpa_f, "ours_fwd_bwd": ours_fb, "sdpa_fwd_bwd": sdpa_fb},
                      args.reps, args.iters)
        emit(what="attention", B=B, S=S, H=H, **{k: round(v, 4) for k, v in r.items()})


def rows(args):
    from baton_b200.ops import load
    C = load()
    B, S = 128, 65
    for D in (192, 384):
        rows_ = B * S
        torch.manual_seed(0)
        x, r, dy, ds = (torch.randn(rows_, D, device=DEV).to(BF16) for _ in range(4))
        y, s, dsum = (torch.empty(rows_, D, device=DEV, dtype=BF16) for _ in range(3))
        gamma, beta = torch.ones(D, device=DEV), torch.zeros(D, device=DEV)
        dg, db = torch.zeros(D, device=DEV), torch.zeros(D, device=DEV)
        mean, rstd = torch.empty(rows_, device=DEV), torch.empty(rows_, device=DEV)
        z = torch.randn(B, S - 1, D, device=DEV).to(BF16)
        cls, bias, pos = torch.randn(D, device=DEV), torch.randn(D, device=DEV), torch.randn(S, D, device=DEV)
        tok = torch.empty(B, S, D, device=DEV, dtype=BF16)
        dz = torch.empty_like(z)
        gc, gb, gp = torch.zeros(D, device=DEV), torch.zeros(D, device=DEV), torch.zeros(S, D, device=DEV)

        def addln():
            C.layernorm_sum_fwd(x, r, y, s, gamma, beta, mean, rstd, rows_, D, 1e-6)
            C.layernorm_sum_bwd(s, dy, ds, dsum, gamma, mean, rstd, dg, db, rows_, D)

        def tokens():
            C.vit_tokens_fwd(z, cls, bias, pos, tok, B, S, D)
            C.vit_tokens_bwd(tok, dz, gc, gb, gp, B, S, D)

        res = alternate({"add_ln_fwd_bwd": addln, "tokens_fwd_bwd": tokens}, args.reps, args.iters)
        # bytes each pair must move at least: add+LN reads x, r, dy, ds, s and writes y, s, dsum; tokens read z and
        # dtok and write tok and dz (bf16)
        gbs = {"add_ln_fwd_bwd": 8 * rows_ * D * 2, "tokens_fwd_bwd": 4 * rows_ * D * 2}
        emit(what="rows", shape=[rows_, D], **{k: round(v, 4) for k, v in res.items()},
             **{k + "_GBps": round(gbs[k] / (v * 1e-3) / 1e9, 1) for k, v in res.items()})


def rounds(args):
    from baton_b200.data import dirichlet_label_shards, image_shard
    from baton_b200.models import resnet18, vit_tiny
    from baton_b200.parallel.engine import FederatedEngine
    spec = dirichlet_label_shards(1, 10, 4096, 0.5, 0)[0]
    X, y = image_shard(spec, seed=0, dtype=BF16)
    X, y = X.to(DEV), y.to(DEV)
    engines = {}
    for name, ctor, lr in (("vit_tiny", vit_tiny, 0.01), ("resnet18", resnet18, 0.05)):
        torch.manual_seed(0)
        engines[name] = FederatedEngine(ctor(10), DEV, backend="fused", lr=lr, batch_size=128, momentum=0.9)
        engines[name].run_round((X, y), n_epoch=1)          # warm-up: capture and first replay
        engines[name].sync()
    torch.cuda.synchronize()
    times = {k: [] for k in engines}
    loss = {}
    for _ in range(args.rounds):
        for k, eng in engines.items():
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            res = eng.run_round((X, y), n_epoch=1)
            eng.sync()
            e.record()
            e.synchronize()
            times[k].append(s.elapsed_time(e))
            loss[k] = res.loss_history[-1]
    for k, v in times.items():
        emit(what="round", model=k, samples=4096, batch=128, round_ms=round(statistics.median(v), 2),
             samples_per_s=round(4096 / (statistics.median(v) * 1e-3)), last_loss=round(loss[k], 4))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("vit_bench needs a CUDA device")
    name, pl = card()
    emit(what="card", name=name, power_limit=pl)
    attention(args)
    rows(args)
    rounds(args)


if __name__ == "__main__":
    main()
