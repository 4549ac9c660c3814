"""Secure aggregation: what the encode + mask kernel costs, and what a secure round costs against a plain fp32-wire one.

* encode kernel alone (``F.secagg_encode``): CUDA events over 50 launches for 0..7 peers on the ResNet-18 arena
  (11.18 M parameters, 44.7 MB of theta) and the BERT-base arena, theta - global read (8 B / element) and the ring words
  written (4 B / element); the bandwidth is those bytes over the kernel time.
* rounds (1 GPU): the ResNet-18 flagship round (4096 samples, batch 128, 1 local epoch, SGD lr 0.05) with the plain
  fp32 wire against ``secure_agg=True``, device-timed, in alternating blocks (the ``clip_bench.py`` method).
* multi-GPU rounds are not measured by this script; it reports them as such.

    python scripts/secagg_bench.py [--reps 5] [--rounds-per-rep 3]

Reads the card name, power limit and SM clock in the same run and prints one JSON line."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from fedprox_bench import card  # noqa: E402


def rounds(torch, engines, shard, args):
    """Median device time of a round per engine, over alternating blocks of ``rounds_per_rep`` rounds."""
    def block(eng, m):
        ms = []
        for _ in range(m):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            eng.run_round(shard, n_epoch=1, read_loss=False)
            eng.sync()
            e1.record()
            e1.synchronize()
            ms.append(e0.elapsed_time(e1))
        return sorted(ms)[len(ms) // 2]

    keys = list(engines)
    for k in keys:
        block(engines[k], 2)                           # capture + warm-up
    reps = {k: [] for k in keys}
    for r in range(args.reps):
        for k in (keys if r % 2 == 0 else keys[::-1]):
            reps[k].append(block(engines[k], args.rounds_per_rep))
            print("rep {} {:<6} {:.3f} ms/round".format(r, k, reps[k][-1]), flush=True)
    out = {"round_ms_" + k: sorted(v)[len(v) // 2] for k, v in reps.items()}
    out.update({"round_ms_range_" + k: [min(v), max(v)] for k, v in reps.items()})
    return out


def encode_kernel(torch, dev, n, peers, launches=50):
    from baton_b200.ops import functional as F
    theta = torch.randn(n, device=dev) * 1e-2
    glob = torch.zeros(n, device=dev)
    out = torch.empty(n, dtype=torch.int32, device=dev)
    sat = torch.zeros(1, dtype=torch.int64, device=dev)
    keys = [[(p * 8 + j) * 2654435761 & 0xFFFFFFFF for j in range(8)] for p in range(peers)]
    signs = [1 if p % 2 else -1 for p in range(peers)]

    def go():
        F.secagg_encode(theta, glob, 0.5, 64.0, 24, keys, signs, (1, 0, 0), 0, out, sat)

    for _ in range(5):
        go()
    per = []
    for _ in range(5):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(launches):
            go()
        e1.record()
        e1.synchronize()
        per.append(e0.elapsed_time(e1) * 1e3 / launches)
    us = sorted(per)[len(per) // 2]
    return {"peers": peers, "us": round(us, 1), "us_range": [round(min(per), 1), round(max(per), 1)],
            "GBps": round(12 * n / us / 1e3, 1)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--rounds-per-rep", type=int, default=3)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("secagg_bench.py measures on a CUDA device; none is available")
    dev = torch.device("cuda:0")
    out = card()
    from baton_b200.data import dirichlet_label_shards, image_shard
    from baton_b200.models import bert_base, resnet18
    from baton_b200.parallel.arena import ParamArena
    from baton_b200.parallel.engine import FederatedEngine
    for name, mk in (("resnet18", lambda: resnet18(10)), ("bert_base", lambda: bert_base(2))):
        n = ParamArena(mk(), torch.device("cpu")).n
        out["encode_" + name] = {"n": n, "by_peers": [encode_kernel(torch, dev, n, p) for p in range(8)]}
        print(name, out["encode_" + name], flush=True)
    spec = dirichlet_label_shards(1, 10, 4096, alpha=0.5, seed=11)[0]
    X, y = image_shard(spec, seed=3, dtype=torch.bfloat16)
    engines = {}
    for k, on in (("fp32", False), ("secure", True)):
        torch.manual_seed(0)
        engines[k] = FederatedEngine(resnet18(10), dev, backend="fused", lr=0.05, batch_size=128, n_ctas=132, seed=5,
                                     wire_dtype="fp32", secure_agg=on)
    r = rounds(torch, engines, (X.to(dev), y.to(dev)), args)
    r["overhead"] = r["round_ms_secure"] / r["round_ms_fp32"] - 1.0
    r["saturated"] = engines["secure"].last_secagg_saturation()
    r["config"] = "resnet18, 4096 samples, batch 128, 1 local epoch, sgd lr 0.05"
    out["rounds_resnet18_1gpu"] = r
    out["rounds_multi_gpu"] = "not measured"
    out["sm_clock_after"] = card().get("sm_clock")
    print(json.dumps(out))


if __name__ == "__main__":
    main()
