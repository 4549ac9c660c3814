"""LoRA on the GPU: the down projection, the rank-R epilogue of the base GEMM (forward and data-gradient forms) and
the adapter gradients against float64 -- exact on small-integer operands with a power-of-two scale, bounded on
full-mantissa bf16 -- their determinism, and a LoRA BERT trained by the graphed trainer and the fused engine."""
import copy

import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
BF16 = torch.bfloat16

# (output slices, targeted slices): packed q/v, packed q/k/v, a single-slice ffn_in
PATTERNS = {"qv": (3, (True, False, True)), "qkv": (3, (True, True, True)), "ffn_in": (1, (True,))}


def _operands(M, K, ds, n_sl, T, r, exact, seed):
    g = torch.Generator().manual_seed(seed)
    if exact:       # integers: every product and sum below is exact in fp32, U and V exact in bf16
        mk = lambda *s: torch.randint(-1, 2, s, generator=g).double()
    else:
        mk = lambda *s: torch.randn(*s, generator=g).to(BF16).double()
    x, w, b = mk(M, K), mk(n_sl * ds, K), mk(n_sl * ds)
    a, bb, dy = mk(T * r, K), mk(T * ds, r), mk(M, n_sl * ds)
    return x, w, b, a, bb, dy


def _slots(targets):
    slot, t = [-1, -1, -1], 0
    for i, on in enumerate(targets):
        if on:
            slot[i], t = t, t + 1
    return slot, t


def _check(out, ref, exact, what):
    out = out.double().cpu()
    assert torch.isfinite(out).all(), what + ": unwritten (NaN) elements"
    if exact:
        assert torch.equal(out, ref), what
    else:
        err = float((out - ref).abs().max() / ref.abs().max())
        assert err < 2e-2, (what, err)


@pytest.mark.parametrize("exact", [True, False], ids=["exact", "bounded"])
@pytest.mark.parametrize("pattern", list(PATTERNS))
@pytest.mark.parametrize("r", [8, 16, 32, 64])
def test_lora_kernels_against_float64(r, pattern, exact):
    from baton_b200.ops import functional as F
    n_sl, targets = PATTERNS[pattern]
    slot, T = _slots(targets)
    if T * r > 192:
        pytest.skip("more than 192 ranks in one layer")
    M, K, ds = 200, 64, 96             # M is not a multiple of the 128-row tile
    s = 0.5
    x, w, b, a, bb, dy = _operands(M, K, ds, n_sl, T, r, exact, seed=r + 7 * n_sl + T)
    d = lambda t: t.to(device=DEV, dtype=BF16).contiguous()
    # down projection into a NaN-guarded buffer
    u = torch.full((M, T * r), float("nan"), dtype=BF16, device=DEV)
    F.lora_down(d(x), d(a), T=1, rs=T * r, kt=K, xoff=(0,), w_ts=0, wsj=K, wsk=1, out=u)
    u_ref = x @ a.t()
    _check(u, u_ref.to(BF16).double(), True if exact else False, "U = X A^T")
    u64 = u.double().cpu()            # the kernel's bf16 U is the operand of what follows
    # forward epilogue form, fp32 output
    y = torch.full((M, n_sl * ds), float("nan"), dtype=torch.float32, device=DEV)
    F.gemm_lora(d(x), d(w), dict(u=u, f=d(bb), fs_n=r, fs_j=1, rs=r, ds=ds, slot=slot, s=s),
                bias=b.float().to(DEV), out_dtype=torch.float32, out=y)
    y_ref = x @ w.t() + b
    for i in range(n_sl):
        if slot[i] >= 0:
            t = slot[i]
            y_ref[:, i * ds:(i + 1) * ds] += s * (u64[:, t * r:(t + 1) * r] @ bb[t * ds:(t + 1) * ds].t())
    _check(y, y_ref, exact, "forward epilogue")
    # V = dY' B per targeted slice, then the data-gradient form dX = dY W + s V A
    sl = sorted((i for i in range(3) if slot[i] >= 0), key=lambda i: slot[i])
    v = torch.full((M, T * r), float("nan"), dtype=BF16, device=DEV)
    F.lora_down(d(dy), d(bb), T=T, rs=r, kt=ds, xoff=[i * ds for i in sl], w_ts=ds * r, wsj=1, wsk=r, out=v)
    v_ref = torch.cat([dy[:, i * ds:(i + 1) * ds] @ bb[slot[i] * ds:(slot[i] + 1) * ds] for i in sl], 1)
    _check(v, v_ref.to(BF16).double(), exact, "V = dY' B")
    v64 = v.double().cpu()
    dx = torch.full((M, K), float("nan"), dtype=torch.float32, device=DEV)
    F.gemm_lora(d(dy), d(w), dict(u=v, f=d(a), fs_n=1, fs_j=K, rs=T * r, ds=K, slot=(0, -1, -1), s=s), b_mn=True,
                out_dtype=torch.float32, out=dx)
    _check(dx, dy @ w + s * (v64 @ a), exact, "data-gradient epilogue")
    # adapter gradients, accumulated onto a known value
    ga = torch.full((T * r, K), 3.0, dtype=torch.float32, device=DEV)
    F.lora_grad_(d(x), v, ga, NA=K, NB=T * r, lo=(0,), qo=(0,), osa=1, osb=K, out_ts=0, s=s)
    _check(ga - 3.0, s * (v64.t() @ x), exact, "dA = s V^T X")
    gb = torch.full((T * ds, r), 3.0, dtype=torch.float32, device=DEV)
    F.lora_grad_(d(dy), u, gb, NA=ds, NB=r, lo=[i * ds for i in sl], qo=[slot[i] * r for i in sl], osa=r, osb=1,
                 out_ts=ds * r, s=s)
    gb_ref = torch.cat([s * (dy[:, i * ds:(i + 1) * ds].t() @ u64[:, slot[i] * r:(slot[i] + 1) * r]) for i in sl], 0)
    _check(gb - 3.0, gb_ref, exact, "dB = s dY'^T U")


def test_adapter_gradients_are_deterministic_eager_and_graphed():
    from baton_b200.ops import functional as F
    torch.manual_seed(0)
    M, K, R = 4096 + 77, 768, 16
    x = torch.randn(M, K, device=DEV).to(BF16)
    v = torch.randn(M, R, device=DEV).to(BF16)
    outs = []
    for _ in range(2):
        g = torch.zeros(R, K, device=DEV)
        F.lora_grad_(x, v, g, NA=K, NB=R, lo=(0,), qo=(0,), osa=1, osb=K, out_ts=0, s=2.0)
        outs.append(g)
    g = torch.zeros(R, K, device=DEV)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        F.lora_grad_(x, v, torch.zeros(R, K, device=DEV), NA=K, NB=R, lo=(0,), qo=(0,), osa=1, osb=K, out_ts=0, s=2.0)
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        F.lora_grad_(x, v, g, NA=K, NB=R, lo=(0,), qo=(0,), osa=1, osb=K, out_ts=0, s=2.0)
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(outs[0], outs[1]) and torch.equal(outs[0], g)


def _tokens(n, seed):
    g = torch.Generator().manual_seed(seed)
    X = torch.randint(0, 1024, (n, 64), generator=g)
    return X, (X[:, :4].sum(1) % 2)


def test_bert_tiny_lora_epoch_keeps_frozen_weights_and_tracks_cpu():
    from baton_b200.models.bert import LoraConfig, bert_tiny
    from baton_b200.ops import functional as F
    from baton_b200.ops import nn as bnn
    from baton_b200.parallel.arena import ParamArena
    from baton_b200.train import GraphedLocalSGD, PortableLocalSGD
    torch.manual_seed(3)
    m = bert_tiny(2, lora=LoraConfig(8, 16, targets=("query", "value")))
    with torch.no_grad():
        for n, p in m.named_parameters():
            if n.endswith("lora_B"):
                p.normal_(0, 0.02)
    cpu = copy.deepcopy(m)
    arena = ParamArena(m, DEV)
    lo, hi = arena.frozen_range
    theta0, shadow0 = arena.theta[lo:hi].clone(), arena.theta_bf16[lo:hi].clone()
    X, y = _tokens(16, seed=1)          # one batch per epoch: the CPU and GPU trainers see the same batches
    # one backward: the only weight-gradient GEMM is the classifier's; layer 0 (input from the frozen embeddings) runs
    # no data gradient, layer 1's goes through the LoRA epilogue form
    calls = {"wgrad": 0, "lora_dgrad": 0}
    gemm, gemm_lora = F.gemm, F.gemm_lora

    def count_gemm(a, b, **kw):
        calls["wgrad"] += bool(kw.get("a_mn") and kw.get("b_mn"))
        return gemm(a, b, **kw)

    def count_lora(a, b, lora, **kw):
        calls["lora_dgrad"] += bool(kw.get("b_mn"))
        return gemm_lora(a, b, lora, **kw)
    F.gemm, F.gemm_lora = count_gemm, count_lora
    try:
        loss, _ = bnn.cross_entropy(m(X[:16].to(DEV)), y[:16].to(DEV))
        loss.backward()
        torch.cuda.synchronize()
    finally:
        F.gemm, F.gemm_lora = gemm, gemm_lora
    assert calls == {"wgrad": 1, "lora_dgrad": 1}, calls
    arena.grad.zero_()
    tr = GraphedLocalSGD(m, arena, loss="ce")
    m._graphed_trainer = tr
    torch.manual_seed(11)
    tr.run(X.to(DEV), y.to(DEV), n_epoch=3, lr=0.05, batch_size=16)
    torch.cuda.synchronize()
    assert torch.equal(arena.theta[lo:hi], theta0) and torch.equal(arena.theta_bf16[lo:hi], shadow0)
    # the CPU trainer on the same batches (fp32 throughout): the adapters move the same way within bf16 rounding
    carena = ParamArena(cpu, torch.device("cpu"))
    torch.manual_seed(11)
    init = cpu.lora_state_dict()
    PortableLocalSGD(cpu, carena, loss="ce").run(X, y, n_epoch=3, lr=0.05, batch_size=16)
    gpu_sd, cpu_sd = m.lora_state_dict(), cpu.lora_state_dict()
    for k in gpu_sd:
        step_gpu, step_cpu = gpu_sd[k].cpu() - init[k], cpu_sd[k] - init[k]
        err = float((step_gpu - step_cpu).norm() / (step_cpu.norm() + 1e-12))
        assert err < 0.2, (k, err)      # bf16 activations against fp32


@pytest.mark.parametrize("wire", ["bf16", "fp8"])
def test_engine_round_uploads_adapters_only(wire):
    from baton_b200.models.bert import LoraConfig, bert_tiny
    from baton_b200.parallel.engine import FederatedEngine
    torch.manual_seed(4)
    m = bert_tiny(2, lora=LoraConfig(8, 16))
    eng = FederatedEngine(m, DEV, backend="fused", lr=1e-3, batch_size=16, optimizer="adamw", wire_dtype=wire)
    a = eng.arena
    lo, hi = a.frozen_range
    frozen0 = a.theta[lo:hi].clone()
    X, y = _tokens(64, seed=2)
    res = eng.run_round((X.to(DEV), y.to(DEV)), n_epoch=2)
    assert all(v == v for v in res.loss_history)
    n = a.n - (hi - lo)
    assert eng.last_upload_bytes() == (2 * n if wire == "bf16" else n + (n + 31) // 32)
    assert torch.equal(a.theta[lo:hi], frozen0)
    assert torch.equal(a.theta[:lo], a.global_w[:lo])
    eng.evaluate((X.to(DEV), y.to(DEV)))
