"""Small run of every kernel family for compute-sanitizer (memcheck / racecheck / synccheck):
   compute-sanitizer --tool memcheck python scripts/sanitize_smoke.py"""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from baton_b200.models import bert_tiny, resnet18  # noqa: E402
from baton_b200.ops import functional as F  # noqa: E402
from baton_b200.ops import nn as bnn  # noqa: E402
from baton_b200.parallel.arena import ParamArena  # noqa: E402
from baton_b200.parallel.fedavg import FedAvgSession  # noqa: E402

dev = torch.device("cuda:0")
torch.manual_seed(0)
BF16 = torch.bfloat16
# GEMM: all majors, cluster split-K, atomic split-K, batched, fp8
A = torch.randn(256, 512, device=dev).to(BF16)
B = torch.randn(192, 512, device=dev).to(BF16)
for amn in (False, True):
    for bmn in (False, True):
        F.gemm(A.t().contiguous() if amn else A, B.t().contiguous() if bmn else B, a_mn=amn, b_mn=bmn)
F.gemm(torch.randn(128, 2048, device=dev).to(BF16), torch.randn(256, 2048, device=dev).to(BF16), split_k=-4, force_bn=64)
F.gemm(A.t().contiguous(), B.t().contiguous(), a_mn=True, b_mn=True, out=torch.zeros(512, 512, device=dev)[:256, :192].contiguous(), accumulate=True, split_k=3)
qa, sa = F.quant_mx_rows(A)
qb, sb = F.quant_mx_rows(B)
F.gemm_fp8(qa, sa, qb, sb, 512)
F.quant_mx_cols(A)
# ResNet-18 step (conv, BN, pool, loss, SGD) and BERT-tiny step (attention, LN, embedding)
m = resnet18(10)
arena = ParamArena(m, dev, momentum=True)
m.build_workspace(dev)
x = torch.randn(16, 32, 32, 3, device=dev).to(BF16)
y = torch.randint(0, 10, (16,), device=dev)
loss, _ = bnn.cross_entropy(m(x), y)
loss.backward()
bnn.WGRAD.join()
hyper = torch.tensor([0.05, 0.9, 1e-4, 0.0], device=dev)
F.fused_sgd(arena.theta[: arena.n_param], arena.grad, hyper, arena.momentum, arena.theta_bf16[: arena.n_param])
# round 2: the hand-scheduled step (implicit-GEMM conv fwd / dgrad / wgrad, cluster BatchNorm backward with two-piece
# gradients, byte-argmax max-pool, one-launch classifier head), the optimizer emitting the upload copy (K4), and the
# collective with arrival flags consumed by the gated first convolution (K3)
sess = FedAvgSession(arena, n_ctas=8, tile_flags=True)
sess.gate_first_conv(m.conv1)
m.explicit_step(x, y)
sess.arm_prepack(16.0)
F.fused_sgd(arena.theta[: arena.n_param], arena.grad, hyper, arena.momentum, arena.theta_bf16[: arena.n_param],
            pack=sess.pack_spec())
sess.aggregate(my_n=16.0, prepacked=True, on_side_stream=True)
m.explicit_step(x, y)            # staging kernel + conv1 GEMM acquire the flags while the collective is in flight
sess.join()
sess.aggregate(my_n=16.0)
# fused attention (S = 128, d = 64)
qkv = torch.randn(2 * 128, 3 * 2 * 64, device=dev).to(BF16).requires_grad_(True)
bnn.attention(qkv, 2, 128, 2, 64).sum().backward()
b = bert_tiny(3)
ab = ParamArena(b, dev)
ids = torch.randint(0, 1024, (4, 64), device=dev)
loss, _ = bnn.cross_entropy(b(ids), torch.randint(0, 3, (4,), device=dev))
loss.backward()
bnn.WGRAD.join()
torch.cuda.synchronize()
print("sanitize smoke done")
