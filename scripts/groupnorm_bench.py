"""GroupNorm: what the kernels cost on ResNet-18's shapes, and what GroupNorm costs a flagship round.

* kernels, on every GroupNorm input of ResNet-18 at batch 128 on 32x32 images (bf16 NHWC, G = 2, ReLU on, no residual):
  - ``gn_fwd`` (statistics + apply in one launch) and ``gn_bwd`` (one dy piece, dgamma / dbeta accumulated);
  - torch's ``F.group_norm`` + ReLU on the same channels_last bf16 tensors (forward, including the layout copy torch
    makes), and ``native_group_norm_backward`` after the ReLU mask on the contiguous copy (backward);
  - the BatchNorm kernels they replace: ``bn_apply`` (the statistics come from the conv GEMM's epilogue) and the
    BatchNorm backward (``bn_bwd_cluster`` where it applies, else reduce + apply), accumulating into fp32 gradient
    buffers as the arena does.
  Every operation's outputs are allocated once; 200 calls are captured into ONE CUDA graph and the graph is replayed
  between CUDA events, so the host is out of the timed loop.  The time per call is therefore the device time of the
  operation inside a captured sequence, as in the training step, including the graph's launch gap between nodes;
  ``launch_floor_us`` is the same measurement for the smallest possible ``gn_fwd`` (one 1x1x8 sample), the per-node
  floor.  Achieved bandwidth is the bytes the operation must move (forward: read z, write y; backward: read z, y, dy,
  write dz) over that time, against the H100 SXM's 3.35 TB/s.  The tensors (at most 4 MB each) stay in the 50 MB L2.
  ``per_step_us`` adds up the per-call times over the 20 norm layers of a ResNet-18 step (1, 4, 5, 5 and 5 of the five
  shapes), forward and backward; for BatchNorm the real stem runs the fused ``bn_relu_maxpool`` pair instead.
* rounds: device-timed rounds of the flagship configuration (1 GPU, ResNet-18, 4096 Dirichlet(0.5) samples, batch 128,
  1 local epoch, SGD lr 0.05) with ``norm="batch"`` and ``norm="group"`` in alternating blocks, the ``clip_bench.py``
  method; medians and ranges.

    python scripts/groupnorm_bench.py [--reps 5] [--rounds-per-rep 3]

Reads the card name, power limit and SM clock in the same run and prints one JSON line."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from fedprox_bench import card  # noqa: E402

SHAPES = [(16, 16, 64), (8, 8, 64), (4, 4, 128), (2, 2, 256), (1, 1, 512)]
HBM_BPS = 3.35e12


def _graph_time(torch, fn, launches=200, reps=5):
    """Median and range of the device time per call of ``fn``: ``launches`` calls in one captured graph, replayed between
    CUDA events."""
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):          # warm-up outside the capture (kernel attributes, lazy initialisation)
        for _ in range(3):
            fn()
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        for _ in range(launches):
            fn()
    graph.replay()
    torch.cuda.synchronize()
    per = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        graph.replay()
        e1.record()
        e1.synchronize()
        per.append(e0.elapsed_time(e1) * 1e3 / launches)
    del graph
    return round(sorted(per)[len(per) // 2], 2), [round(min(per), 2), round(max(per), 2)]


LAYERS = [1, 4, 5, 5, 5]      # norm layers of a ResNet-18 step on each of SHAPES


def kernels(torch, dev, n=128, groups=2):
    from torch.nn import functional as TF
    from baton_b200.ops import functional as F
    L = F.load()
    bf = torch.bfloat16
    out = {"shapes": []}
    z1 = torch.ones(1, 1, 1, 8, device=dev, dtype=bf)
    p1, y1, s1 = torch.ones(8, device=dev), torch.empty_like(z1), torch.empty(1, device=dev)
    out["launch_floor_us"] = _graph_time(torch, lambda: L.gn_fwd(z1, None, y1, p1, p1, s1, s1, 1, 1e-5, True, None))[0]
    for h, w, c in SHAPES:
        g = torch.Generator(device=dev).manual_seed(0)
        z = (torch.randn(n, h, w, c, device=dev, generator=g) + 1).to(bf)
        dy = torch.randn(n, h, w, c, device=dev, generator=g).to(bf)
        gamma, beta = torch.ones(c, device=dev), torch.zeros(c, device=dev)
        dgamma, dbeta = torch.zeros(c, device=dev), torch.zeros(c, device=dev)
        y, dz = torch.empty_like(z), torch.empty_like(z)
        mean, rstd = torch.empty(n, groups, device=dev), torch.empty(n, groups, device=dev)
        work = F.gn_work(n, c, groups, dev)
        L.gn_fwd(z, None, y, gamma, beta, mean, rstd, groups, 1e-5, True, work)
        elem, rows = n * h * w * c, n * h * w
        row = {"shape": [n, h, w, c], "groups": groups}
        row["gn_fwd_us"], row["gn_fwd_range"] = _graph_time(
            torch, lambda: L.gn_fwd(z, None, y, gamma, beta, mean, rstd, groups, 1e-5, True, work))
        row["gn_bwd_us"], row["gn_bwd_range"] = _graph_time(
            torch, lambda: L.gn_bwd(z, y, dy, None, dz, None, gamma, mean, rstd, dgamma, dbeta, groups, True, work))
        row["gn_fwd_TBps"] = round(4 * elem / row["gn_fwd_us"] / 1e6, 3)
        row["gn_bwd_TBps"] = round(8 * elem / row["gn_bwd_us"] / 1e6, 3)
        row["gn_fwd_share_of_hbm"] = round(4 * elem / HBM_BPS * 1e6 / row["gn_fwd_us"], 3)
        row["gn_bwd_share_of_hbm"] = round(8 * elem / HBM_BPS * 1e6 / row["gn_bwd_us"], 3)
        # torch on the same bf16 channels_last data (NCHW view of the NHWC tensor)
        aten = torch.ops.aten
        zt, dyt = z.permute(0, 3, 1, 2), dy.permute(0, 3, 1, 2)
        gt, bt = gamma.to(bf), beta.to(bf)
        try:
            # forward through F.group_norm, which brings the channels_last tensor into the layout its kernel takes (that
            # copy is part of torch's cost); backward through the aten kernel on that contiguous layout
            row["torch_fwd_us"] = _graph_time(torch, lambda: torch.relu(TF.group_norm(zt, groups, gt, bt, 1e-5)))[0]
            zt, dyt = zt.contiguous(), dyt.contiguous()
            yt, mt, rt = aten.native_group_norm(zt, gt, bt, n, c, h * w, groups, 1e-5)
            yt = torch.relu(yt)
            row["torch_bwd_us"] = _graph_time(torch, lambda: aten.native_group_norm_backward(
                aten.threshold_backward(dyt, yt, 0), zt, mt, rt, gt, n, c, h * w, groups, [True, True, True]))[0]
        except RuntimeError as exc:          # recorded, not hidden: the JSON says what torch could not run
            row["torch_error"] = str(exc).splitlines()[0]
        # the BatchNorm kernels of the same layer, gradients accumulated into fp32 buffers like the arena's
        ybn, dx = torch.empty_like(z), torch.empty_like(z)
        sums = torch.zeros(4 * c, device=dev)
        rm, rv = torch.zeros(c, device=dev), torch.ones(c, device=dev)
        smean, srstd = torch.empty(c, device=dev), torch.empty(c, device=dev)
        L.bn_stats(z, sums[: 2 * c], rows, c)
        apply = lambda: L.bn_apply(z, None, ybn, sums[: 2 * c], gamma, beta, rm, rv, smean, srstd, None, rows, c,  # noqa: E731
                                   1e-5, 0.1, True, True)
        apply()
        row["bn_apply_us"] = _graph_time(torch, apply)[0]
        cluster = L.bn_bwd_cluster(z, ybn, dy, None, dx, None, gamma, smean, srstd, dgamma, dbeta, rows, c, True, 16)
        if cluster:
            bwd = lambda: L.bn_bwd_cluster(z, ybn, dy, None, dx, None, gamma, smean, srstd, dgamma, dbeta,  # noqa: E731
                                           rows, c, True, 16)
        else:
            def bwd():
                L.bn_bwd_reduce(z, ybn, dy, smean, srstd, sums[2 * c:], rows, c, True)
                L.bn_bwd_apply(z, ybn, dy, dx, None, gamma, smean, srstd, sums[2 * c:], dgamma, dbeta, rows, c, True)
        row["bn_bwd_path"] = "cluster" if cluster else "reduce+apply"
        row["bn_bwd_us"] = _graph_time(torch, bwd)[0]
        out["shapes"].append(row)
        print(row, flush=True)
    rs = out["shapes"]
    out["per_step_us"] = {
        "group_fwd": round(sum(k * r["gn_fwd_us"] for k, r in zip(LAYERS, rs)), 1),
        "group_bwd": round(sum(k * r["gn_bwd_us"] for k, r in zip(LAYERS, rs)), 1),
        "batch_fwd": round(sum(k * r["bn_apply_us"] for k, r in zip(LAYERS, rs)), 1),
        "batch_bwd": round(sum(k * r["bn_bwd_us"] for k, r in zip(LAYERS, rs)), 1)}
    return out


def round_block(torch, engines, shard, args):
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=shard[0].device)

    def block(k, m):
        ms = []
        for _ in range(m):
            flush.zero_()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            engines[k].run_round(shard, n_epoch=1, read_loss=False)
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
        out["round_ms_" + k] = round(sorted(v)[len(v) // 2], 3)
        out["round_ms_range_" + k] = [round(min(v), 3), round(max(v), 3)]
    out["group_over_batch"] = round(out["round_ms_group"] / out["round_ms_batch"] - 1.0, 4)
    return out


def flagship(args, torch, dev):
    from baton_b200.data import dirichlet_label_shards, image_shard
    from baton_b200.models import resnet18
    from baton_b200.parallel.engine import FederatedEngine
    spec = dirichlet_label_shards(1, 10, 4096, alpha=0.5, seed=11)[0]
    X, y = image_shard(spec, seed=3, dtype=torch.bfloat16)
    engines = {}
    for k in ("batch", "group"):
        torch.manual_seed(0)
        engines[k] = FederatedEngine(resnet18(10, norm=k), dev, backend="fused", lr=0.05, batch_size=128, n_ctas=132,
                                     seed=5)
    out = round_block(torch, engines, (X.to(dev), y.to(dev)), args)
    out["kernels_per_step"] = {k: e.trainer.n_kernels_per_step for k, e in engines.items()}
    out["config"] = "resnet18, 4096 samples, batch 128 (32 steps), 1 local epoch, sgd lr 0.05, G = 2"
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--rounds-per-rep", type=int, default=3)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("groupnorm_bench.py measures on a CUDA device; none is available")
    dev = torch.device("cuda:0")
    out = card()
    out["kernels_resnet18_b128"] = kernels(torch, dev)
    out["rounds_resnet18"] = flagship(args, torch, dev)
    out["sm_clock_after"] = card().get("sm_clock")
    print(json.dumps(out))


if __name__ == "__main__":
    main()
