"""In-graph kernel timeline of the captured local-SGD epoch (needs the trace build of the extension):

    BATON_BUILD_TRACE=1 python -m baton_b200.build_ext          # once, here or on the GPU box
    BATON_TRACE=1 python scripts/trace_step.py --model resnet18 --out gpurun_out/trace_r18.txt

Prints (a) the per-kernel-type share of the critical path over one replayed epoch and (b) the ordered kernel list
of one steady-state step with each kernel's slot (time until the next kernel's dependencies were satisfied)."""
import argparse
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from baton_b200.data import ShardSpec, image_shard, token_shard  # noqa: E402
from baton_b200.models import bert_base, resnet18, resnet50  # noqa: E402
from baton_b200.parallel.arena import ParamArena  # noqa: E402
from baton_b200.train import GraphedLocalSGD  # noqa: E402
from baton_b200.utils.trace import KernelTrace  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--model", default="resnet18")
ap.add_argument("--steps", type=int, default=8)
ap.add_argument("--batch-size", type=int, default=128)
ap.add_argument("--out", default="")
ap.add_argument("--points", default="", help="kernel name: print the intra-kernel TRACE_POINT stamps of its first 3 launches")
args = ap.parse_args()
dev = torch.device("cuda:0")
torch.manual_seed(0)
is_bert = args.model == "bert_base"
m = bert_base(2) if is_bert else (resnet18(10) if args.model == "resnet18" else resnet50(10))
arena = ParamArena(m, dev)
if not is_bert:
    m.build_workspace(dev)
tr = GraphedLocalSGD(m, arena, loss="ce", use_graph=True)
n = args.batch_size * args.steps
if is_bert:
    X, y = token_shard(ShardSpec(0, torch.full((2,), 0.5), n), seq_len=128)
else:
    X, y = image_shard(ShardSpec(0, torch.full((10,), 0.1), n), dtype=torch.bfloat16)
X, y = X.to(dev), y.to(dev)
for _ in range(2):
    tr.run(X, y, n_epoch=1, lr=0.05, batch_size=args.batch_size)      # capture + warm replay
torch.cuda.synchronize()
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
e0.record()
tr.run(X, y, n_epoch=1, lr=0.05, batch_size=args.batch_size, return_device=True)
e1.record()
torch.cuda.synchronize()
untraced_ms = e0.elapsed_time(e1)
kt = KernelTrace(capacity=1 << 17, device=dev)
ok = kt.start()
e0.record()
tr.run(X, y, n_epoch=1, lr=0.05, batch_size=args.batch_size, return_device=True)
e1.record()
kt.stop()
lines = ["# model {} batch {} steps/epoch {}  kernels/step {}  epoch {:.3f} ms untraced, {:.3f} ms traced (trace build active: {})".format(
    args.model, args.batch_size, args.steps, tr.n_kernels_per_step, untraced_ms, e0.elapsed_time(e1), ok)]
rows = kt.timeline()
lines += kt.summary()
# one steady-state step: from the (steps//2)-th optimizer kernel to the next
sgd = [i for i, r in enumerate(rows) if r["name"] in ("fused_sgd_kernel", "fused_sgd_segments_kernel")]
if len(sgd) >= 3:
    a, b = sgd[len(sgd) // 2 - 1] + 1, sgd[len(sgd) // 2] + 1
    lines.append("# one step ({} kernels, {:.1f} us): t_us since step start | slot us | resident-before-deps us | kernel".format(
        b - a, (rows[b - 1]["t_ns"] + rows[b - 1]["slot_ns"] - rows[a]["t_ns"]) / 1e3))
    t0 = rows[a]["t_ns"]
    for r in rows[a:b]:
        lines.append("{:9.2f} {:7.2f} {:7.2f}  {}".format((r["t_ns"] - t0) / 1e3, r["slot_ns"] / 1e3, r["early_ns"] / 1e3, r["name"]))
if args.points:
    pts = kt.points()
    shown = 0
    for i, (t, lab) in enumerate(pts):
        if lab.startswith("> " + args.points) and shown < 3 and i > len(pts) // 3:
            shown += 1
            lines.append("# intra-kernel points of {} (us since its dependencies completed); next kernel start closes the list".format(args.points))
            prev_end = max((tt for tt, ll in pts[:i] if ll.startswith("> ")), default=t)
            lines.append("   previous kernel's dependencies done {:8.2f} us earlier".format((t - prev_end) / 1e3))
            for tt, ll in pts[i + 1: i + 40]:
                lines.append("{:9.2f}  {}".format((tt - t) / 1e3, ll))
                if ll.startswith("> "):
                    break
text = "\n".join(lines)
print(text)
if args.out:
    with open(args.out, "w") as f:
        f.write(text + "\n")
