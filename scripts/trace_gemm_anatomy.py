"""Where does a latency-bound conv GEMM spend its ~3-7 us?  Intra-kernel %globaltimer stamps (trace build) of the fixed
GEMM kernel inside a captured chain conv -> bn_apply -> conv ..., printed as offsets from the moment the kernel's
dependencies completed.   BATON_TRACE=1 python scripts/trace_gemm_anatomy.py"""
import collections
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from baton_b200.ops import functional as F  # noqa: E402
from baton_b200.ops import load  # noqa: E402
from baton_b200.utils.trace import KernelTrace  # noqa: E402

dev = torch.device("cuda:0")
BF16 = torch.bfloat16
C = load()
REPS = 12


def chain(name, n, h, cin, cout, k, stride, pad, stats=True):
    x = torch.randn(n, h, h, cin, device=dev).to(BF16)
    w = (torch.randn(cout, k * k * cin, device=dev) * 0.05).to(BF16)
    ho = F.conv_out_size(h, k, stride, pad)
    M = n * ho * ho
    y = torch.empty(M, cout, device=dev, dtype=BF16)
    z = torch.empty(M, cout, device=dev, dtype=BF16)
    ws = torch.zeros(REPS, 4 * cout, device=dev)
    gamma, beta = torch.ones(cout, device=dev), torch.zeros(cout, device=dev)
    rm, rv = torch.zeros(cout, device=dev), torch.ones(cout, device=dev)
    sm, sr = torch.empty(cout, device=dev), torch.empty(cout, device=dev)

    def run():
        ws.zero_()
        for i in range(REPS):
            assert C.conv_igemm_fwd(x, w, y, k, k, stride, pad, ho, ho, 1, 64, ws[i][: 2 * cout] if stats else None)
            C.bn_apply(y, None, z, ws[i][: 2 * cout], gamma, beta, rm, rv, sm, sr, None, M, cout, 1e-5, 0.1, True, True)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        run(); run()
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        run()
    g.replay(); torch.cuda.synchronize()
    kt = KernelTrace(capacity=1 << 14, device=dev)
    kt.start()
    g.replay()
    kt.stop()
    pts = kt.points()
    # group: for every GEMM start, offsets of the following points until the next kernel start
    acc = collections.defaultdict(list)
    order = []
    i = 0
    while i < len(pts):
        t0, lab = pts[i]
        if lab.startswith("> gemm_bf16_fixed"):
            j = i + 1
            prev_end = None
            while j < len(pts) and not pts[j][1].startswith("> "):
                if pts[j][1].startswith("    . "):
                    key = pts[j][1].strip(" .")
                    acc[key].append((pts[j][0] - t0) / 1e3)
                    if key not in order:
                        order.append(key)
                j += 1
            if j < len(pts):
                acc["next kernel (bn_apply) dependencies done"].append((pts[j][0] - t0) / 1e3)
        i += 1
    print("{}  M={} N={} K={} stats={}  ({} launches)".format(name, M, cout, k * k * cin, stats, len(acc.get(order[0], [])) if order else 0))
    for key in order + ["next kernel (bn_apply) dependencies done"]:
        v = sorted(acc[key])
        if v:
            print("   +{:6.2f} us (median)  {}".format(v[len(v) // 2], key))


chain("1x1 s2 downsample (1 k-tile)", 128, 8, 64, 128, 1, 2, 0)
chain("layer1 3x3 (9 k-tiles)", 128, 8, 64, 64, 3, 1, 1)
chain("layer1 3x3 (9 k-tiles), no stats", 128, 8, 64, 64, 3, 1, 1, stats=False)
