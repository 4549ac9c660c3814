"""BERT tier: strided-batched wgmma GEMM, fused attention core, embedding, and the BERT encoder
against fp32 PyTorch references."""
import math
import os

import pytest
import torch

pytestmark = pytest.mark.gpu
BF16 = torch.bfloat16


def _rel(a, b):
    a, b = a.detach().float(), b.detach().float()
    return float((a - b).abs().max() / (b.abs().max() + 1e-6))


def test_attention_core_forward_backward():
    from baton_b200.ops import nn as bnn
    torch.manual_seed(0)
    dev = torch.device("cuda:0")
    # the last two shapes have >= 296 (batch x head x tile) problems: persistent batched kernel
    for (B, S, H, dh) in [(4, 128, 12, 64), (2, 64, 2, 64), (3, 256, 4, 32), (32, 128, 12, 64), (8, 256, 12, 64)]:
        D = H * dh
        qkv = (torch.randn(B * S, 3 * D, device=dev) * 0.5).to(BF16).requires_grad_(True)
        out = bnn.attention(qkv, B, S, H, dh)
        ref_in = qkv.detach().float().requires_grad_(True)
        q, k, v = (t.reshape(B, S, H, dh).transpose(1, 2) for t in ref_in.split(D, dim=-1))
        p = torch.softmax(q @ k.transpose(-1, -2) / math.sqrt(dh), dim=-1)
        ref = (p @ v).transpose(1, 2).reshape(B * S, D)
        assert out.shape == ref.shape and _rel(out, ref) < 2e-2, (B, S, H, dh, _rel(out, ref))
        g = torch.randn_like(out)
        out.backward(g)
        ref.backward(g.float())
        assert _rel(qkv.grad, ref_in.grad) < 4e-2, (B, S, H, dh, _rel(qkv.grad, ref_in.grad))


def test_embedding_forward_backward():
    from baton_b200.ops import nn as bnn
    torch.manual_seed(1)
    dev = torch.device("cuda:0")
    emb = bnn.Embedding(1000, 128).to(dev)
    ids = torch.randint(0, 1000, (16, 32), device=dev)
    out = emb(ids)
    assert torch.equal(out, emb.weight.detach().to(BF16)[ids.reshape(-1)])
    g = torch.randn_like(out)
    out.backward(g)
    ref = torch.zeros(1000, 128, device=dev).index_add_(0, ids.reshape(-1), g.float())
    assert _rel(emb.weight.grad, ref) < 1e-3


def test_bert_tiny_matches_fp32_reference_and_trains():
    from baton_b200.models import bert_tiny
    from baton_b200.ops import nn as bnn
    from baton_b200.parallel.arena import ParamArena
    from baton_b200.train import GraphedLocalSGD
    torch.manual_seed(2)
    dev = torch.device("cuda:0")
    m = bert_tiny(3)
    ref = bert_tiny(3)
    ref.load_state_dict(m.state_dict())
    arena = ParamArena(m, dev)
    ids = torch.randint(0, 1024, (8, 64))
    y = torch.randint(0, 3, (8,))
    logits = m(ids.to(dev))
    ref_logits = ref(ids)                                   # CPU fp32 path of the same module
    assert _rel(logits.cpu(), ref_logits) < 5e-2
    loss, _ = bnn.cross_entropy(logits, y.to(dev))
    loss.backward()
    torch.nn.functional.cross_entropy(ref_logits, y).backward()
    cos = torch.nn.functional.cosine_similarity
    refp = dict(ref.named_parameters())
    sims = {n: float(cos(p.grad.flatten().cpu(), refp[n].grad.flatten(), dim=0)) for n, p in m.named_parameters()
            if refp[n].grad is not None and float(refp[n].grad.abs().max()) > 0}
    worst = min(sims, key=sims.get)
    assert sum(sims.values()) / len(sims) > 0.97 and sims[worst] > 0.85, (worst, sims[worst])
    arena.grad.zero_()
    # CUDA-graphed local SGD on token shards
    X = torch.randint(0, 1024, (256, 64), device=dev)
    yy = (X[:, :8].sum(1) % 3).to(dev)
    tr = GraphedLocalSGD(m, arena, loss="ce")
    m._graphed_trainer = tr
    hist = m.train(X, yy, n_epoch=8, lr=0.05, batch_size=32)
    assert hist[-1] < hist[0], hist


def test_fused_attention_forward_and_backward_match_masked_multi_kernel_path():
    from baton_b200.ops import nn as bnn
    torch.manual_seed(0)
    dev = torch.device("cuda:0")
    B, S, H, dh = 8, 128, 12, 64
    D = H * dh
    qkv = (torch.randn(B * S, 3 * D, device=dev) * 0.5).to(BF16)
    outs = []
    # a mask sends forward and backward down the multi-kernel path; adding a bf16 zero to the scores is exact
    for mask_bias in (torch.zeros(B, S, device=dev), None):
        x = qkv.clone().requires_grad_(True)
        out = bnn.attention(x, B, S, H, dh, mask_bias=mask_bias)
        g = torch.ones_like(out)
        out.backward(g)
        outs.append((out.detach().float(), x.grad.float()))
    assert _rel(outs[1][0], outs[0][0]) < 2e-2
    assert _rel(outs[1][1], outs[0][1]) < 3e-2
