"""Dropout of BERT training on the H100: the dropout forms of the LayerNorm, softmax, elementwise and fused attention
kernels against float64 with the host mask (data/dropout.py), the masks bit for bit, p = 0 as the model without
dropout, the model against a float64 reference, graph replay across rounds and clients, and engine rounds.

Windows: with p = 0.5 (s = 2, exact) the masked operands are exact, so the checks are the bf16 output rounding plus
fp32 accumulation (rtol 2^-7 of the row scale); with p = 0.1 and full-mantissa operands the same windows hold."""
import math

import numpy as np
import pytest
import torch

from baton_b200.data.augment import augment_key
from baton_b200.data.dropout import DropoutRun, dropout_keep, scale

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
BF = torch.bfloat16
F64 = torch.float64
KEY, STREAM = augment_key(21), (3 << 32) | 5
ROW_CS = [64, 128, 256, 512, 768, 1024, 100]          # every ROW_DISPATCH pair, and the scalar kernel (C % 8 != 0)


@pytest.fixture(scope="module")
def C_():
    from baton_b200.ops._ext import load
    return load()


def _run(site_count=8, steps=4, epoch=1, step=2):
    run = DropoutRun()
    run.begin(KEY, STREAM, steps, 3, site_count)
    words = torch.tensor([epoch, STREAM & 0xFFFFFFFF, STREAM >> 32], dtype=torch.int64).to(torch.int32).to(DEV)
    run.at(epoch, step, words)
    return run


def _keep(run, site, n, p):
    return torch.from_numpy(dropout_keep(KEY, STREAM, site, run.t, n, p)).to(DEV)


def _data(shape, dyadic, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    if dyadic:
        x = torch.randint(1, 8, shape, device=DEV, generator=g).to(torch.float32) * 0.25
        x = x * (torch.randint(0, 2, shape, device=DEV, generator=g) * 2 - 1)
    else:
        x = torch.randn(shape, device=DEV, generator=g) + 0.05
    return x.to(BF)


def _close(got, want, tol):
    want = want.to(F64)
    err = (got.to(F64) - want).abs().max().item()
    ref = want.abs().max().item()
    assert err <= tol * max(ref, 1e-30), (err, ref)


def _ln_ref(v, g, b, eps=1e-12):
    mu = v.mean(-1, keepdim=True)
    var = ((v - mu) ** 2).mean(-1, keepdim=True)
    return (v - mu) / torch.sqrt(var + eps) * g + b, mu, var


@pytest.mark.parametrize("p", [0.5, 0.1])
@pytest.mark.parametrize("C", ROW_CS)
@pytest.mark.parametrize("mode", [1, 2])
def test_layernorm_dropout_forms(C_, mode, C, p):
    rows = 77
    run = _run()
    site = 2 if mode == 1 else 0
    da = run.kernel_args(site, p)
    x, r, dy = _data((rows, C), p == 0.5, 1), _data((rows, C), p == 0.5, 2), _data((rows, C), p == 0.5, 3)
    gam = (torch.randint(1, 4, (C,), device=DEV) * 0.5).float()
    bet = (torch.randint(-2, 3, (C,), device=DEV) * 0.25).float()
    keep = _keep(run, site, rows * C, p).view(rows, C)
    s = scale(p)
    y = torch.full_like(x, float("nan"))
    pre = torch.full_like(x, float("nan")) if mode == 1 else None
    mean, rstd = torch.empty(rows, device=DEV), torch.empty(rows, device=DEV)
    C_.layernorm_drop_fwd(x, r, y, pre, gam, bet, mean, rstd, rows, C, 1e-12, mode, *da)
    xd, rd, gd, bd = x.to(F64), r.to(F64), gam.to(F64), bet.to(F64)
    m = keep.to(F64) * torch.tensor(s, dtype=torch.float32).to(F64)
    v = xd * m + rd if mode == 1 else xd + rd
    yr, mu, var = _ln_ref(v, gd, bd)
    if mode == 2:
        yr = yr * m
    _close(y, yr, 2 ** -6)
    if mode == 2:
        assert bool((y[~keep] == 0).all())
    if mode == 1:          # fp32(x s), plus the residual in fp32, rounded once to bf16
        s32 = torch.tensor(s, dtype=torch.float32, device=DEV)
        assert torch.equal(pre, torch.where(keep, x.float() * s32, torch.zeros_like(x.float())).add(r.float()).to(BF))
    # backward against the kernel's own statistics
    pre_in = pre if mode == 1 else (x.float() + r.float()).to(BF)
    dx = torch.full_like(x, float("nan"))
    dxd = torch.full_like(x, float("nan")) if mode == 1 else None
    dg, db = torch.zeros(C, device=DEV), torch.zeros(C, device=DEV)
    C_.layernorm_drop_bwd(pre_in, dy, dx, dxd, gam, mean, rstd, dg, db, rows, C, mode, *da)
    h = (pre_in.to(F64) - mean.to(F64)[:, None]) * rstd.to(F64)[:, None]
    g = dy.to(F64) * (m if mode == 2 else 1.0)
    gw = g * gd
    dpre = rstd.to(F64)[:, None] * (gw - gw.mean(-1, keepdim=True) - h * (gw * h).mean(-1, keepdim=True))
    _close(dx, dpre, 2 ** -6)
    _close(dg, (g * h).sum(0), 2 ** -12)
    _close(db, g.sum(0), 2 ** -12)
    if mode == 1:
        _close(dxd, dpre * m, 2 ** -6)
        assert bool((dxd[~keep] == 0).all())


@pytest.mark.parametrize("p", [0.5, 0.1])
@pytest.mark.parametrize("C", ROW_CS)
def test_softmax_dropout_forms(C_, C, p):
    rows = 93
    run = _run()
    da = run.kernel_args(4, p)
    x, dy = _data((rows, C), p == 0.5, 4), _data((rows, C), p == 0.5, 5)
    keep = _keep(run, 4, rows * C, p).view(rows, C)
    m = keep.to(F64) * float(np.float32(scale(p)))
    y, yd, dx = (torch.full_like(x, float("nan")) for _ in range(3))
    C_.softmax_drop_fwd(x, y, yd, rows, C, 0.5, *da)
    P = torch.softmax(x.to(F64) * 0.5, -1)
    _close(y, P, 2 ** -7)
    _close(yd, P * m, 2 ** -7)
    assert torch.equal(yd != 0, keep)                            # P > 0 everywhere: the zeros are the mask
    C_.softmax_drop_bwd(y, dy, dx, rows, C, 0.5, *da)
    Pd = y.to(F64)
    g = dy.to(F64) * m
    _close(dx, 0.5 * Pd * (g - (Pd * g).sum(-1, keepdim=True)), 2 ** -6)


def test_elementwise_dropout(C_):
    run = _run()
    for n, p in ((32 * 768, 0.1), (1001, 0.5)):
        da = run.kernel_args(7, p)
        x = _data((n,), False, 6)
        y = torch.full_like(x, float("nan"))
        C_.dropout(x, y, *da)
        keep = _keep(run, 7, n, p)
        want = torch.where(keep, (x.float() * np.float32(scale(p))).to(BF), torch.zeros_like(x))
        assert torch.equal(y, want)


def _attn_ref(qkv, B, S, H, dh, keep, s, dout):
    D = H * dh
    q, k, v = (t.to(F64).reshape(B, S, H, dh).transpose(1, 2).requires_grad_(True)
               for t in qkv.split(D, dim=-1))
    P = torch.softmax(q @ k.transpose(-1, -2) / math.sqrt(dh), -1)
    o = ((P * keep.view(B, H, S, S).to(F64) * s) @ v).transpose(1, 2).reshape(B * S, D)
    o.backward(dout.to(F64))
    dq, dk, dv = (t.grad.transpose(1, 2).reshape(B * S, D) for t in (q, k, v))
    return o.detach(), torch.cat([dq, dk, dv], -1), P.detach()


@pytest.mark.parametrize("B", [1, 8, 32])
def test_fused_attention_dropout_against_float64(C_, B):
    H, S, dh, p = 12, 128, 64, 0.1
    D = H * dh
    run = _run()
    da = run.kernel_args(1, p)
    qkv = (torch.randn(B * S, 3 * D, device=DEV) * 0.5).to(BF)
    dout = torch.randn(B * S, D, device=DEV).to(BF)
    out = torch.full((B * S, D), float("nan"), dtype=BF, device=DEV)
    probs = torch.full((B * H * S, S), float("nan"), dtype=BF, device=DEV)
    dqkv = torch.full_like(qkv, float("nan"))
    sc = 1.0 / math.sqrt(dh)
    assert C_.attention_drop_fwd(qkv, out, probs, B, S, H, dh, sc, *da)
    assert C_.attention_drop_bwd(qkv, dout, probs, dqkv, B, S, H, dh, sc, *da)
    keep = _keep(run, 1, B * H * S * S, p)
    o, dq, P = _attn_ref(qkv, B, S, H, dh, keep, float(np.float32(scale(p))), dout)
    _close(probs, P.reshape(B * H * S, S), 2 ** -7)               # the saved probabilities are undropped
    _close(out, o, 2 ** -5)
    _close(dqkv, dq, 2 ** -4)


def test_fused_and_multi_kernel_paths_drop_the_same_probabilities():
    from baton_b200.ops import nn as bnn
    B, H, S, dh, p = 4, 12, 128, 64, 0.5
    D = H * dh
    run = _run()
    qkv = (torch.randn(B * S, 3 * D, device=DEV) * 0.5).to(BF)
    dout = torch.randn(B * S, D, device=DEV).to(BF)
    outs = []
    for mask in (None, torch.zeros(B, S, device=DEV)):
        x = qkv.clone().requires_grad_(True)
        o = bnn.attention(x, B, S, H, dh, mask_bias=mask, drop=(run, 1, p))
        o.backward(dout)
        outs.append((o.detach().float(), x.grad.float()))
    (o1, g1), (o2, g2) = outs
    assert (o1 - o2).abs().max().item() <= 2 ** -5 * o2.abs().max().item()
    assert (g1 - g2).abs().max().item() <= 2 ** -4 * g2.abs().max().item()
    # the zero pattern of the dropped probabilities equals the host mask in the multi-kernel path
    from baton_b200.ops._ext import load
    sc = torch.full((B * H * S, S), 0.25, dtype=BF, device=DEV)
    P, Pd = torch.empty_like(sc), torch.empty_like(sc)
    load().softmax_drop_fwd(sc, P, Pd, B * H * S, S, 1.0, *run.kernel_args(1, p))
    assert torch.equal(Pd != 0, _keep(run, 1, B * H * S * S, p).view(B * H * S, S))


def _tiny(p=0.0, **kw):
    from baton_b200.models.bert import BertConfig, BertForSequenceClassification
    torch.manual_seed(0)
    return BertForSequenceClassification(BertConfig(
        vocab_size=1024, hidden_size=128, num_hidden_layers=2, num_attention_heads=2, intermediate_size=512,
        max_position_embeddings=128, hidden_dropout_prob=p, attention_probs_dropout_prob=p, **kw), name="bert_tiny")


def _tokens(n, S=128, seed=0):
    g = torch.Generator().manual_seed(seed)
    return torch.randint(0, 1024, (n, S), generator=g), torch.randint(0, 2, (n,), generator=g)


def test_p0_is_the_model_without_dropout():
    from baton_b200.models import bert_tiny
    from baton_b200.ops._ext import launch_counts
    from baton_b200.ops import nn as bnn
    ids, y = _tokens(8)
    res = []
    torch.manual_seed(0)
    plain = bert_tiny(2)                                         # the same initialisation as _tiny's
    for m in (plain, _tiny(0.0, classifier_dropout=0.0)):
        m.to(DEV).train()
        c0 = launch_counts()
        out = m(ids.to(DEV))
        loss, _ = bnn.cross_entropy(out, y.to(DEV))
        loss.backward()
        torch.cuda.synchronize()
        res.append((out.detach(), [p.grad.clone() for p in m.parameters()], launch_counts() - c0))
    (o1, g1, k1), (o2, g2, k2) = res
    assert torch.equal(o1, o2) and k1 == k2
    # the LayerNorm and embedding backward accumulate with fp32 atomics, so gradients agree to their summation order
    for a, b in zip(g1, g2):
        assert (a - b).norm() <= 1e-5 * b.norm() + 1e-12


def test_bert_tiny_against_float64_reference_with_host_masks():
    """The CUDA model in train mode against the CPU model (float64, dropout_reference masks) on the same run state."""
    from baton_b200.ops import nn as bnn
    ids, y = _tokens(4, seed=2)
    cpu = _tiny(0.1)
    gpu = _tiny(0.1)
    gpu.load_state_dict(cpu.state_dict())
    cpu = cpu.double()
    gpu.to(DEV).train()
    cpu.train()
    for m, dev in ((gpu, DEV), (cpu, None)):
        run = m.dropout_run
        run.begin(KEY, STREAM, 4, 2, m.n_dropout_sites)
        words = torch.tensor([1, STREAM & 0xFFFFFFFF, STREAM >> 32], dtype=torch.int64).to(torch.int32).to(DEV)
        run.at(1, 3, words)
    out = gpu(ids.to(DEV))
    loss, _ = bnn.cross_entropy(out, y.to(DEV))
    loss.backward()
    ref = cpu(ids)
    lref = torch.nn.functional.cross_entropy(ref, y)
    lref.backward()
    _close(out.float().cpu(), ref.detach(), 2 ** -4)
    for (name, pg), pc in zip(gpu.named_parameters(), cpu.parameters()):
        if pc.grad is None or pc.grad.abs().max() == 0:
            continue
        err = (pg.grad.double().cpu() - pc.grad).norm().item()
        assert err <= 0.1 * pc.grad.norm().item(), name
    for m in (gpu, cpu):
        m.dropout_run.end()


def _init_theta():
    from baton_b200.parallel.arena import ParamArena
    return ParamArena(_tiny(0.1), DEV).theta.clone()


def test_graphed_equals_eager_and_replays_for_new_rounds_and_clients():
    from baton_b200.parallel.arena import ParamArena
    from baton_b200.train import GraphedLocalSGD
    X, y = _tokens(40, seed=3)
    X, y = X.to(DEV), y.to(DEV)
    thetas = []
    for use_graph in (True, False):
        m = _tiny(0.1)
        arena = ParamArena(m, DEV)
        tr = GraphedLocalSGD(m, arena, loss="ce", use_graph=use_graph)
        torch.manual_seed(7)
        tr.run(X, y, n_epoch=2, lr=0.01, batch_size=16, augment_seed=5, augment_stream=11)
        thetas.append(arena.theta.clone())
        if use_graph:
            graphs = len(tr._graphs)
            before = arena.theta.clone()
            torch.manual_seed(7)
            tr.run(X, y, n_epoch=2, lr=0.01, batch_size=16, augment_seed=5, augment_stream=(1 << 32) | 2)
            assert len(tr._graphs) == graphs                     # a new round / client replays the captured epoch
            assert not torch.equal(arena.theta, before)
    # the same masks: graphed and eager differ only by the summation order of the fp32-atomic gradient sums
    assert (thetas[0] - thetas[1]).norm() <= 1e-4 * (thetas[1] - _init_theta()).norm()


def test_second_stream_draws_its_own_masks():
    from baton_b200.parallel.arena import ParamArena
    from baton_b200.train import GraphedLocalSGD
    X, y = _tokens(32, seed=4)
    X, y = X.to(DEV), y.to(DEV)
    res = {}
    for stream in (1, 2, 1):
        m = _tiny(0.1)
        arena = ParamArena(m, DEV)
        tr = GraphedLocalSGD(m, arena, loss="ce")
        torch.manual_seed(3)
        tr.run(X, y, n_epoch=1, lr=0.05, batch_size=16, augment_seed=5, augment_stream=stream)
        res.setdefault(stream, []).append(arena.theta.clone())
    base = _init_theta()
    same = (res[1][0] - res[1][1]).norm()
    other = (res[1][0] - res[2][0]).norm()
    assert same <= 1e-4 * (res[1][0] - base).norm() and other > 100 * same


@pytest.mark.parametrize("opts", [dict(optimizer="adamw", lr=1e-3), dict(max_grad_norm=0.5), dict(wire_dtype="fp8")],
                         ids=["adamw", "clip", "fp8-wire"])
def test_engine_rounds_with_dropout_and_evaluate_independent_of_p(opts):
    from baton_b200.parallel.engine import FederatedEngine
    opts = dict(opts)
    X, y = _tokens(64, seed=5)
    X, y = X.to(DEV), y.to(DEV)
    kw = dict(backend="fused", lr=0.01, batch_size=16, seed=3)
    kw.update(opts)
    engines = []
    for p in (0.1, 0.0):
        m = _tiny(p)
        engines.append(FederatedEngine(m, DEV, **kw))
    a, b = engines
    for _ in range(2):
        res = a.run_round((X, y), n_epoch=1)
    assert all(math.isfinite(v) for v in res.loss_history)
    b.model.load_state_dict(a.model.state_dict())
    b.arena.commit_global()
    ea, eb = a.evaluate((X, y)), b.evaluate((X, y))
    assert ea == eb
