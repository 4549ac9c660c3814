"""Top-k uploads (parallel/compress.py) on one GPU: the selection + compaction per client and the fused collective alone,
plain against top-k.  Blocks of the variants alternate, CUDA events time each block, and the median block is reported.

    python scripts/topk_bench.py [--out topk_bench.json]

Bytes per selection (what the passes must move, from shapes): the first pass reads theta, global_w and e and writes u
(16 B per element), the next two histogram passes and the count pass read u (4 B each), the write pass reads u (4 B)
and writes the k entries (2 B offset + the value) and the row pointers; zeroing the kept residual entries adds 4 B per
entry.  Bandwidth is those bytes over the measured time, against the H100 SXM data-sheet 3.35 TB/s."""
import argparse
import json
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from baton_b200.parallel.compress import GRANULE, TopKConfig  # noqa: E402

DEV = "cuda:0"
ARENAS = {"resnet18": 11_190_272, "bert_base": 109_483_008}     # float elements, whole granules
RATIOS = (0.001, 0.01, 0.1)
PEAK = 3.35e12


def _time_blocks(fns, iters, blocks):
    """fns: name -> callable; alternating blocks of `iters` calls; median ms per call."""
    ts = {k: [] for k in fns}
    for _ in range(blocks):
        for k, fn in fns.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(iters):
                fn()
            e1.record()
            torch.cuda.synchronize()
            ts[k].append(e0.elapsed_time(e1) / iters)
    return {k: statistics.median(v) for k, v in ts.items()}


def selection(iters, blocks):
    from baton_b200.ops import functional as F
    out = []
    for name, n in ARENAS.items():
        gen = torch.Generator(device=DEV).manual_seed(0)
        g = torch.randn(n, device=DEV, generator=gen)
        theta = g + torch.randn(n, device=DEV, generator=gen) * 1e-3
        e = torch.randn(n, device=DEV, generator=gen) * 1e-4
        work = F.topk_work(n, DEV)
        fns, meta = {}, {}
        for r in RATIOS:
            k = TopKConfig(r).k(n)
            rowptr = torch.zeros(n // GRANULE + 1, dtype=torch.int32, device=DEV)
            off = torch.zeros(k, dtype=torch.int16, device=DEV)
            val = torch.zeros(k, dtype=torch.bfloat16, device=DEV)

            def fn(k=k, rowptr=rowptr, off=off, val=val):
                F.topk_pack(theta, g, e, k, work, rowptr.data_ptr(), off.data_ptr(), val.data_ptr(), ef=True,
                            wire_fp32=False, cap=k)
            fn()
            fns[r] = fn
            meta[r] = 16 * n + 4 * n * 4 + k * (2 + 2 + 4) + 4 * (n // GRANULE + 1)
        torch.cuda.synchronize()
        ms = _time_blocks(fns, iters, blocks)
        for r in RATIOS:
            t = ms[r] * 1e-3
            out.append({"arena": name, "n": n, "ratio": r, "k": TopKConfig(r).k(n), "us": ms[r] * 1e3,
                        "bytes": meta[r], "gbps": meta[r] / t / 1e9, "share_of_3.35TBps": meta[r] / t / PEAK})
            print("select+compact {:9s} ratio {:5}: {:8.1f} us, {:6.0f} GB/s ({:.0%} of 3.35 TB/s)".format(
                name, r, ms[r] * 1e3, meta[r] / t / 1e9, meta[r] / t / PEAK), flush=True)
        del g, theta, e, work
        torch.cuda.empty_cache()
    return out


def collective(iters, blocks):
    from baton_b200.models import resnet18
    from baton_b200.parallel.arena import ParamArena
    from baton_b200.parallel.fedavg import FedAvgSession
    torch.manual_seed(0)
    sess, arenas = {}, {}
    for key in ("plain",) + RATIOS:
        a = ParamArena(resnet18(10), DEV)
        a.theta.add_(torch.randn_like(a.theta) * 1e-3)
        arenas[key] = a
        kw = {} if key == "plain" else {"topk": TopKConfig(key, error_feedback=False)}
        sess[key] = FedAvgSession(a, wire_dtype="bf16", mode="delta", nvls=False, **kw)
    fns = {}
    for key, s in sess.items():
        def fn(s=s, key=key):
            a = arenas[key]
            a.theta.add_(1e-6)           # a fresh update every round (a round makes theta the global model)
            if key != "plain":
                s.pack_topk()
            s.aggregate(my_n=1.0)
        fns[key] = fn
        fn()

    # the collective alone: the lists the timed rounds above left in both wire halves are sent again
    only = {}
    for key, s in sess.items():
        def fn2(s=s, key=key):
            arenas[key].theta.add_(1e-6)
            if key != "plain":
                s._topk_lists()
                s._packed_epoch = s.epoch
            s.aggregate(my_n=1.0)
        only[key] = fn2
    torch.cuda.synchronize()
    round_ms = _time_blocks({str(k): fns[k] for k in fns}, iters, blocks)
    coll_ms = _time_blocks({str(k): only[k] for k in only}, iters, blocks)
    out = []
    for k in fns:
        out.append({"variant": str(k), "round_with_selection_us": round_ms[str(k)] * 1e3,
                    "collective_us": coll_ms[str(k)] * 1e3})
        print("collective {:6s}: {:7.1f} us alone, {:7.1f} us with the selection".format(
            str(k), coll_ms[str(k)] * 1e3, round_ms[str(k)] * 1e3), flush=True)
    for s in sess.values():
        s.check()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--blocks", type=int, default=7)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("topk_bench.py measures on a GPU; none is visible")
    props = torch.cuda.get_device_properties(0)
    import subprocess
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       stdout=subprocess.PIPE, text=True).stdout.strip()
    print("device:", props.name, "|", q, flush=True)
    res = {"device": props.name, "nvidia_smi": q, "selection": selection(args.iters, args.blocks),
           "collective_resnet18_bf16": collective(args.iters, args.blocks)}
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
