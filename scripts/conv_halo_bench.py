"""ResNet-18 layer1 convolution (3x3, stride 1, 64 -> 64 channels, 8x8 maps, batch 128) forward and input gradient:
im2col-mode implicit GEMM vs the halo-tiled kernel.  As in scripts/mb_layers.py each rep is the GEMM followed by a
full-GPU bn_apply inside a captured graph, so consecutive GEMMs cannot overlap each other the way identical
back-to-back launches do; the bn_apply time alone is measured and subtracted.  The two paths alternate over
repetitions.  Beside each time: the bytes every CTA and every launch pulls through TMA, computed from the shapes.

    python scripts/conv_halo_bench.py [--batch 128] [--reps 5] [--json out.json]
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

BF16 = torch.bfloat16
CH = 64
CHAIN = 20


def tma_bytes(n, h, w, path):
    """(CTAs, bytes per CTA, bytes per launch) the TMA loads of one layer1 GEMM move (fwd and dgrad alike)."""
    m = n * h * w
    if path == "im2col":
        bn = F.pick_bn(m, CH)
        ctas = ((m + 127) // 128) * ((CH + bn - 1) // bn)
        per = 9 * (128 * CH * 2) + 9 * (bn * CH * 2)      # one im2col box per tap + nine weight k-tiles
    else:
        ctas = (m + F.HALO_BM - 1) // F.HALO_BM
        mc = F.halo_cluster(m)
        per = (F.HALO_BM // (h * w)) * (h + 2) * (w + 2) * CH * 2 + 9 * CH * CH * 2 // mc
    return ctas, per, ctas * per


def time_graph(fn, iters=10):
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            fn()
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        fn()
    g.replay()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        g.replay()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1e3 / iters


def gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              stdout=subprocess.PIPE, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return torch.cuda.get_device_name(0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=128)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("conv_halo_bench needs a CUDA device")
    C = load()
    dev = torch.device("cuda:0")
    n, h = args.batch, 8
    m = n * h * h
    x = torch.randn(n, h, h, CH, device=dev).to(BF16)
    w = (torch.randn(CH, 9 * CH, device=dev) * 0.05).to(BF16)
    y = torch.empty(m, CH, device=dev, dtype=BF16)
    z = torch.empty(m, CH, device=dev, dtype=BF16)
    ws = torch.zeros(CHAIN, 4 * CH, device=dev)
    gamma, beta = torch.ones(CH, device=dev), torch.zeros(CH, device=dev)
    rm, rv = torch.zeros(CH, device=dev), torch.ones(CH, device=dev)
    sm, sr = torch.empty(CH, device=dev), torch.empty(CH, device=dev)

    def bn(i):
        C.bn_apply(y, None, z, ws[i][: 2 * CH], gamma, beta, rm, rv, sm, sr, None, m, CH, 1e-5, 0.1, True, True)

    def bn_only():
        for i in range(CHAIN):
            bn(i)

    def chain(kind, path):
        def run():
            ws.zero_()
            for i in range(CHAIN):
                if kind == "fwd":
                    F.conv_igemm_fwd(x, w, 3, 3, 1, 1, col_stats=ws[i][: 2 * CH], out=y, path=path)
                else:
                    F.conv_igemm_dgrad(x, w, (n, h, h, CH), 3, 3, 1, out=y.view(n, h, h, CH), path=path)
                bn(i)
        return run

    times = {(k, p): [] for k in ("fwd", "dgrad") for p in ("im2col", "halo")}
    bn_t = []
    for _ in range(args.reps):
        bn_t.append(time_graph(bn_only) / CHAIN)
        for k in ("fwd", "dgrad"):
            for p in ("im2col", "halo"):
                times[(k, p)].append(time_graph(chain(k, p)) / CHAIN)
    t_bn = statistics.median(bn_t)
    info = gpu_info()
    print("device: {}".format(info))
    print("layer1 3x3/1 64->64, 8x8, batch {} (M = {}); bn_apply alone {:.2f} us".format(n, m, t_bn))
    out = {"device": info, "batch": n, "bn_apply_us": t_bn}
    for k in ("fwd", "dgrad"):
        for p in ("im2col", "halo"):
            ctas, per, tot = tma_bytes(n, h, h, p)
            t = statistics.median(times[(k, p)]) - t_bn
            out["{}_{}_us".format(k, p)] = t
            print("  {:5s} {:6s} {:6.2f} us per GEMM   CTAs {:3d}  TMA {:6.1f} KB per CTA  {:5.2f} MB per launch".format(
                k, p, t, ctas, per / 1024, tot / 2 ** 20))
        gain = 1 - out["{}_halo_us".format(k)] / out["{}_im2col_us".format(k)]
        out["{}_gain".format(k)] = gain
        print("  {:5s} halo vs im2col: {:+.1f} %".format(k, -100 * gain))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
