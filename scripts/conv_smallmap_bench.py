"""ResNet-18 layer3 convolutions at batch 128 (2x2 output maps, 256 output channels), forward and input gradient:
the im2col-mode implicit GEMM (with the cluster split-K the dispatch picks, and with none) vs the image-tile kernel
(`conv_smallmap`) at each cluster size and, where its weight k-tiles fit, at 64 columns per CTA as well as 32.  As
in scripts/conv_halo_wide_bench.py each rep is the GEMM followed by a full-GPU bn_apply inside a captured graph, so
consecutive GEMMs cannot overlap each other; the bn_apply time alone is measured and subtracted.  The paths
alternate over repetitions.  The card's name, power limit and SM clock are read in the same run.

    python scripts/conv_smallmap_bench.py [--batch 128] [--reps 5] [--paths im2col,im2col-k1,small1,...] [--json f]

Path names: `im2col` (cluster split-K of pick_cluster_k), `im2col-k1`, `small<mc>` (32 columns per CTA, cluster of
mc CTAs along M), `small<mc>-bn64` (64 columns; the stride-2 forward only).
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from baton_b200.ops import functional as F  # noqa: E402
from baton_b200.ops import load  # noqa: E402
from scripts.conv_halo_bench import time_graph  # noqa: E402

BF16 = torch.bfloat16
COUT = 256
CHAIN = 20
# (name, gathered channels, input map, stride, dgrad): layer3.0.conv1 forward (4x4x128 -> 2x2x256, stride 2), and the
# stride-1 256 -> 256 convolutions on 2x2 maps forward and input gradient
SHAPES = [("fwd_s2", 128, 4, 2, False), ("fwd_s1", 256, 2, 1, False), ("dgrad_s1", 256, 2, 1, True)]
PATHS = ["im2col", "im2col-k1", "small1", "small2", "small4", "small8", "small4-bn64"]


def gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                               "--format=csv,noheader"], stdout=subprocess.PIPE, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return torch.cuda.get_device_name(0)


def applies(shape, path):
    return not (path.endswith("-bn64") and shape[0] != "fwd_s2")     # 36 k-tiles of 64 columns do not fit


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=128)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--paths", default=",".join(PATHS))
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    paths = args.paths.split(",")
    if not torch.cuda.is_available():
        raise SystemExit("conv_smallmap_bench needs a CUDA device")
    C = load()
    dev = torch.device("cuda:0")
    n = args.batch
    m = n * 4
    g = torch.Generator(device=dev).manual_seed(0)
    src = {c: torch.randn(n, h, h, c, device=dev, generator=g).to(BF16) for _, c, h, _, _ in SHAPES}
    wts = {c: (torch.randn(COUT, 9 * c, device=dev, generator=g) * 0.05).to(BF16) for _, c, _, _, _ in SHAPES}
    y = torch.empty(m, COUT, device=dev, dtype=BF16)
    z = torch.empty(m, COUT, device=dev, dtype=BF16)
    ws = torch.zeros(CHAIN, 4 * COUT, device=dev)
    gamma, beta = torch.ones(COUT, device=dev), torch.zeros(COUT, device=dev)
    rm, rv = torch.zeros(COUT, device=dev), torch.ones(COUT, device=dev)
    sm, sr = torch.empty(COUT, device=dev), torch.empty(COUT, device=dev)

    def bn(i):
        C.bn_apply(y, None, z, ws[i][: 2 * COUT], gamma, beta, rm, rv, sm, sr, None, m, COUT, 1e-5, 0.1, True, True)

    def bn_only():
        for i in range(CHAIN):
            bn(i)

    def gemm(shape, path, i):
        _, c, h, stride, dgrad = shape
        if path.startswith("small"):
            mc, _, bn = path[5:].partition("-bn")
            kw = dict(path="smallmap", mc=int(mc))
            if bn:
                kw["bn"] = int(bn)
        else:
            kw = dict(path="im2col", cluster_k=1 if path == "im2col-k1" else None)
        if dgrad:
            F.conv_igemm_dgrad(src[c], wts[c], (n, h, h, COUT), 3, 3, 1, out=y.view(n, h, h, COUT), **kw)
        else:
            F.conv_igemm_fwd(src[c], wts[c], 3, 3, stride, 1, col_stats=ws[i][: 2 * COUT], out=y, **kw)

    def chain(shape, path):
        def run():
            ws.zero_()
            for i in range(CHAIN):
                gemm(shape, path, i)
                bn(i)
        return run

    cases = [(s, p) for s in SHAPES for p in paths if applies(s, p)]
    times = {(s[0], p): [] for s, p in cases}
    bn_t = []
    info_before = gpu_info()
    for _ in range(args.reps):
        bn_t.append(time_graph(bn_only) / CHAIN)
        for s, p in cases:
            times[(s[0], p)].append(time_graph(chain(s, p)) / CHAIN)
    t_bn = statistics.median(bn_t)
    info = gpu_info()
    print("device (name, power limit, SM clock, max SM clock): before {} / after {}".format(info_before, info))
    print("layer3 GEMMs, batch {} (M = {}, N = {}); bn_apply alone {:.2f} us; median of {} reps".format(
        n, m, COUT, t_bn, args.reps))
    out = {"device_before": info_before, "device_after": info, "batch": n, "bn_apply_us": t_bn, "reps": args.reps}
    for s, p in cases:
        ts = times[(s[0], p)]
        t = statistics.median(ts) - t_bn
        out["{}_{}_us".format(s[0], p)] = t
        extra = ""
        if p.startswith("im2col"):
            ck = 1 if p == "im2col-k1" else F.pick_cluster_k(m, COUT, 9 * s[1], F.pick_bn(m, COUT))
            extra = "  cluster split-K {}".format(ck)
        print("  {:8s} {:12s} {:6.2f} us per GEMM (spread {:.2f}){}".format(s[0], p, t, max(ts) - min(ts), extra))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
