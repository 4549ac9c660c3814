"""Throughput of evaluating the global model, three ways, alternating:

* ``fused``: ``FederatedEngine.evaluate`` -- one captured graph per pass, every BatchNorm folded into its convolution
  GEMM epilogue (includes the loss, the accuracy and the host read of the result);
* ``graphed``: the ``model.eval()`` forward (GEMM, then ``bn_apply`` in eval mode) captured into one CUDA graph and
  replayed -- the same launch mechanism as ``fused``, so fused against graphed is the effect of the BatchNorm folding;
* ``eager``: the same forward launched op by op -- graphed against eager is the effect of graph replay.

    python scripts/eval_bench.py [--n 10000] [--batch 512] [--reps 5] [--arch resnet18]

Device time from CUDA events around whole passes, after warm-up; prints the card name and power limit read in the
same run, one line per repetition and one JSON summary line."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True, timeout=30).stdout
        name, power = [s.strip() for s in out.strip().splitlines()[0].split(",")]
        return name, power
    except Exception:
        import torch
        return torch.cuda.get_device_name(0), "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=10000)
    ap.add_argument("--batch", type=int, default=512)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--arch", default="resnet18")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("eval_bench.py measures on a CUDA device; none is available")
    from baton_b200 import models
    from baton_b200.data import ShardSpec, holdout_image_shard, image_shard
    from baton_b200.ops._ext import launch_counts
    from baton_b200.parallel.engine import FederatedEngine
    dev = torch.device("cuda:0")
    name, power = card()
    torch.manual_seed(0)
    eng = FederatedEngine(getattr(models, args.arch)(10), dev, backend="fused", lr=0.05, batch_size=128)
    X, y = image_shard(ShardSpec(0, torch.full((10,), 0.1), 1024), noise=0.3, dtype=torch.bfloat16)
    eng.run_round((X.to(dev), y.to(dev)), n_epoch=1)       # non-trivial weights and running statistics
    eng.sync()
    Xe, ye = holdout_image_shard(10, args.n, noise=0.3, dtype=torch.bfloat16)
    Xe, ye = Xe.to(dev), ye.to(dev)
    model = eng.model
    n_batches = (args.n + args.batch - 1) // args.batch

    def fused():
        return eng.evaluate((Xe, ye), batch_size=args.batch)

    def eager():
        torch.nn.Module.train(model, False)
        with torch.no_grad():
            for s in range(0, args.n, args.batch):
                model(Xe[s: s + args.batch])
        torch.nn.Module.train(model, True)

    def timed(fn):
        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        t0.record()
        fn()
        t1.record()
        t1.synchronize()
        return t0.elapsed_time(t1) / 1e3

    res = fused()                     # capture + warm-up
    fused_kernels = sum(eng.trainer.eval_launches.values()) / n_batches
    c0 = launch_counts()
    eager()                           # warm-up, and the launch count of one eager pass
    eager_kernels = sum((launch_counts() - c0).values()) / n_batches
    fused()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        eager()

    def graphed():
        graph.replay()

    graphed()
    rows = {"fused": [], "graphed": [], "eager": []}
    for r in range(args.reps):
        for kind, fn in (("fused", fused), ("graphed", graphed), ("eager", eager)):
            dt = timed(fn)
            rows[kind].append(args.n / dt)
            print("rep {} {:7s} {:9.0f} samples/s".format(r, kind, args.n / dt), flush=True)
    out = {"card": name, "power_limit": power, "arch": args.arch, "n": args.n, "batch": args.batch,
           "fused_kernels_per_batch": fused_kernels, "unfused_kernels_per_batch": eager_kernels,
           "accuracy": res.accuracy, "loss": res.loss}
    for kind, v in rows.items():
        out[kind + "_samples_per_s"] = sorted(v)[len(v) // 2]
        out[kind + "_range"] = [min(v), max(v)]
    out["fold_speedup"] = out["fused_samples_per_s"] / out["graphed_samples_per_s"]
    out["graph_speedup"] = out["graphed_samples_per_s"] / out["eager_samples_per_s"]
    print(json.dumps(out))


if __name__ == "__main__":
    main()
