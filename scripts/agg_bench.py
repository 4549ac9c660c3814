"""Exposed aggregate+broadcast time of one federated round at model sizes of the BASELINE configs:
the fused NVLink kernel (P2P and NVLS variants) vs the NCCL all-reduce baseline, device-timed,
max over ranks.   torchrun --nproc-per-node N scripts/agg_bench.py   (or plain python for N = 1)"""
import json
import os
import sys

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from baton_b200.parallel.arena import ParamArena  # noqa: E402
from baton_b200.parallel.fedavg import FedAvgSession, NcclSession  # noqa: E402

SIZES = {"resnet18": 11_191_242, "resnet50": 25_610_152, "bert_base": 109_482_240}


class Blob(torch.nn.Module):
    def __init__(self, n):
        super().__init__()
        self.w = torch.nn.Parameter(torch.zeros(n))


def main():
    rank = int(os.environ.get("RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    dev = torch.device("cuda", int(os.environ.get("LOCAL_RANK", "0")))
    torch.cuda.set_device(dev)
    if world > 1:
        dist.init_process_group("nccl", device_id=dev)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    rows = []
    ctas_list = [int(x) for x in os.environ.get("AGG_CTAS", "132").split(",")]
    models = os.environ.get("AGG_MODELS", ",".join(SIZES)).split(",")
    wires = os.environ.get("AGG_WIRES", "bf16,fp32,fp8").split(",")
    for name, n in SIZES.items():
        if name not in models:
            continue
        for wire in wires:
            variants = [("nccl", None, 0)] if wire != "fp8" else []      # NCCL has no block-scaled wire
            for c in ctas_list:
                variants += [("fused-p2p", False, c)] + ([("fused-nvls", True, c)] if wire != "fp8" else [])
            for label, nvls, ctas in variants:
                arena = ParamArena(Blob(n), dev)
                arena.theta.normal_()
                if label == "nccl":
                    sess = NcclSession(arena, wire_dtype=wire)
                else:
                    sess = FedAvgSession(arena, wire_dtype=wire, nvls=nvls, n_ctas=ctas)
                    if nvls and not sess.use_nvls:
                        del sess, arena
                        continue
                times = []
                for it in range(8):
                    flush.zero_()
                    if world > 1:
                        dist.barrier()
                    torch.cuda.synchronize()
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    sess.aggregate(my_n=float(100 + rank))
                    e1.record()
                    torch.cuda.synchronize()
                    if it >= 3:
                        times.append(e0.elapsed_time(e1) * 1e3)
                if os.environ.get("AGG_PHASES") == "1" and hasattr(sess, "enable_phase_timing"):
                    sess.enable_phase_timing()
                    sess.aggregate(my_n=float(100 + rank))
                    torch.cuda.synchronize()
                    if rank == 0:
                        print("   phases(us)", {k: {p: round(v, 1) for p, v in d.items()}
                                                for k, d in sess.phase_breakdown_us().items()}, flush=True)
                t = torch.tensor([min(times), sum(times) / len(times)], device=dev, dtype=torch.float64)
                if world > 1:
                    dist.all_reduce(t, op=dist.ReduceOp.MAX)
                wire_bytes = arena.n * (2 if wire == "bf16" else 4) if wire != "fp8" else arena.n + arena.n // 32
                if world > 1:
                    floor = (world - 1) / world * wire_bytes / 450e9 * 1e6     # H100 SXM NVLink, per direction
                    bound = "nvlink450"
                else:
                    fp = arena.n * 4
                    floor = (2 * fp + wire_bytes + 2 * wire_bytes + wire_bytes + fp + 2 * fp + arena.n * 2) / 3.35e12 * 1e6   # H100 SXM HBM3
                    bound = "hbm"
                rows.append({"model": name, "elems": arena.n, "wire": wire, "variant": label, "ctas": ctas,
                             "us_best": float(t[0]), "us_mean": float(t[1]), "floor_us": floor, "bound": bound,
                             "roofline_frac": floor / float(t[0])})
                if rank == 0:
                    r = rows[-1]
                    print("{:10s} {:5s} {:11s} ctas={:3d}  best {:8.1f} us  mean {:8.1f} us  floor({}) {:7.1f} us  frac {:.2f}".format(
                        r["model"], r["wire"], r["variant"], r["ctas"], r["us_best"], r["us_mean"], bound, floor,
                        r["roofline_frac"]), flush=True)
                del sess, arena
                torch.cuda.empty_cache()
    if rank == 0:
        os.makedirs("gpurun_out", exist_ok=True)
        json.dump({"world": world, "rows": rows}, open("gpurun_out/agg_bench_{}gpu.json".format(world), "w"), indent=1)
    if world > 1:
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
