"""ResNet-18 layer2 convolutions at batch 128 (4x4 output maps, 128 output channels), forward and input gradient:
the im2col-mode implicit GEMM (with the cluster split-K the dispatch picks, and with none) vs the wide-channel
halo kernel at each cluster size.  As in scripts/conv_halo_bench.py each rep is the GEMM followed by a full-GPU
bn_apply inside a captured graph, so consecutive GEMMs cannot overlap each other; the bn_apply time alone is
measured and subtracted.  The paths alternate over repetitions.  Beside each time: the bytes every CTA and every
launch pulls through TMA, computed from the shapes.

    python scripts/conv_halo_wide_bench.py [--batch 128] [--reps 5] [--paths im2col,im2col-k1,halo1,...] [--json f]
"""
import argparse
import json
import os
import statistics
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from baton_b200.ops import functional as F  # noqa: E402
from baton_b200.ops import load  # noqa: E402
from scripts.conv_halo_bench import gpu_info, time_graph  # noqa: E402

BF16 = torch.bfloat16
COUT = 128
CHAIN = 20
# (name, gathered channels, input map, stride, dgrad): layer2.0.conv1 forward (8x8x64 -> 4x4x128, stride 2), and the
# stride-1 128 -> 128 convolutions on 4x4 maps forward and input gradient
SHAPES = [("fwd_s2", 64, 8, 2, False), ("fwd_s1", 128, 4, 1, False), ("dgrad_s1", 128, 4, 1, True)]
PATHS = ["im2col", "im2col-k1", "halo1", "halo2", "halo4", "halo8"]


def tma_bytes(n, c, h, stride, dgrad, path):
    """(CTAs, bytes per CTA, bytes per launch) the TMA loads of one of these GEMMs move."""
    ho = h // stride
    m, k = n * ho * ho, 9 * c
    k_tiles = k // 64
    if path.startswith("im2col"):
        bn = F.pick_bn(m, COUT)
        ck = 1 if path == "im2col-k1" else F.pick_cluster_k(m, COUT, k, bn)
        ctas = ((m + 127) // 128) * ((COUT + bn - 1) // bn) * ck
        per = -(-k_tiles // ck) * (128 * 64 * 2 + bn * 64 * 2)       # one im2col box + one weight k-tile per k tile
    else:
        mc = int(path[4:])
        ctas = ((m + F.HALO_BM - 1) // F.HALO_BM) * (COUT // 64)
        hp = stride * (ho - 1) + 3
        per = (F.HALO_BM // (ho * ho)) * hp * hp * c * 2 + k_tiles * 64 * 64 * 2 // mc
    return ctas, per, ctas * per


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=128)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--paths", default=",".join(PATHS))
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    paths = args.paths.split(",")
    if not torch.cuda.is_available():
        raise SystemExit("conv_halo_wide_bench needs a CUDA device")
    C = load()
    dev = torch.device("cuda:0")
    n = args.batch
    m = n * 16
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
        kw = {}
        if path.startswith("halo"):
            kw = dict(path="halo", mc=int(path[4:]))
        else:
            kw = dict(path="im2col", cluster_k=1 if path == "im2col-k1" else None)
        if dgrad:
            F.conv_igemm_dgrad(src[c], wts[c], (n, h, h, c), 3, 3, 1, out=y.view(n, h, h, COUT), **kw)
        else:
            F.conv_igemm_fwd(src[c], wts[c], 3, 3, stride, 1, col_stats=ws[i][: 2 * COUT], out=y, **kw)

    def chain(shape, path):
        def run():
            ws.zero_()
            for i in range(CHAIN):
                gemm(shape, path, i)
                bn(i)
        return run

    times = {(s[0], p): [] for s in SHAPES for p in paths}
    bn_t = []
    for _ in range(args.reps):
        bn_t.append(time_graph(bn_only) / CHAIN)
        for s in SHAPES:
            for p in paths:
                times[(s[0], p)].append(time_graph(chain(s, p)) / CHAIN)
    t_bn = statistics.median(bn_t)
    info = gpu_info()
    print("device: {}".format(info))
    print("layer2 GEMMs, batch {} (M = {}, N = {}); bn_apply alone {:.2f} us; median of {} reps".format(
        n, m, COUT, t_bn, args.reps))
    out = {"device": info, "batch": n, "bn_apply_us": t_bn, "reps": args.reps}
    for s in SHAPES:
        for p in paths:
            ctas, per, tot = tma_bytes(n, s[1], s[2], s[3], s[4], p)
            ts = times[(s[0], p)]
            t = statistics.median(ts) - t_bn
            out["{}_{}_us".format(s[0], p)] = t
            print("  {:8s} {:9s} {:6.2f} us per GEMM (spread {:.2f})  CTAs {:3d}  TMA {:6.1f} KB per CTA  {:5.2f} MB per "
                  "launch".format(s[0], p, t, max(ts) - min(ts), ctas, per / 1024, tot / 2 ** 20))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
