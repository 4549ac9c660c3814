"""Vision Transformer kernels and models on the H100, against float64 and torchvision.

* **Short-S fused attention** (``attention_short_fwd`` / ``_bwd``, csrc/attention.cu), S in {17, 65, 101, 127}, B*H on
  both sides of one wave (132 CTAs):
  - *exact family* (forward): ``scale = fp32(ln 2)``, so ``scale log2(e)`` is 1; small integer Q / K make every score an
    integer and every ``P~`` a power of two, integer V keeps ``P~ V`` and the row sums exact in fp32.  ``out`` and
    ``probs`` must be the nearest-even bf16 of the float64 value, except inside a ``2^-20`` relative band around a
    rounding boundary (the one fp32 reciprocal of the row sum).
  - *bounded family* (bf16 randn at ViT scale): every element of out, dQ, dK, dV within ``2^-7`` of the magnitude of its
    terms (``|P| |V|``, ``|P|^T |dO|``, ...) plus half a bf16 ulp of the value; probs within ``2^-8`` relative.
  - outputs go into NaN-filled buffers with guard elements after them: the rows past the last image and the guard keep
    their bits, the ``probs`` pad columns ``S .. round_up(S, 8) - 1`` are 0, and a second launch gives the same bits.
* **Token kernel**: exact on dyadic inputs, forward and backward (the fp32 sums are exact in any order), accumulating
  into non-zero gradient slots; bitwise-identical across runs and between eager and CUDA-graph replay.
* **Add + LayerNorm writing the sum**: ``s`` exact, ``y`` and ``dsum = LN_bwd(dy) + ds`` within one bf16 ulp plus
  ``2^-14`` of the magnitude of the terms that cancel (``tests/test_gpu_norm_exact.py``'s window), ``dgamma`` / ``dbeta``
  within ``2^-14`` of the sum of their terms' magnitudes.  ``dsum`` is bitwise identical across runs and graph replay;
  ``dgamma`` / ``dbeta`` are accumulated with float atomics as ``layernorm_bwd`` does, so their order is not fixed.
* **erf GELU**: forward and backward within ``2^-8`` relative plus ``2^-20`` absolute of float64.
* **vit_tiny** forward and backward against torchvision's fp32 module on the same weights, and one-GPU
  ``FederatedEngine`` rounds.
"""
import math

import pytest
import torch
from torch.nn import functional as TF

pytestmark = pytest.mark.gpu

BF16 = torch.bfloat16
DEV = torch.device("cuda:0")
GUARD = 1024


@pytest.fixture(scope="module")
def C():
    from baton_b200.ops import load
    return load()


def _nan_buf(n, dtype=BF16):
    buf = torch.full((n + GUARD,), float("nan"), dtype=dtype, device=DEV)
    return buf, buf[:n]


def _sp(S):
    return (S + 7) // 8 * 8


def _ref_attention(qkv, B, S, H, scale, base2=False):
    """float64 probs [B, H, S, S] and out [B*S, D] of packed bf16 qkv"""
    D = H * 64
    q, k, v = (t.double().reshape(B, S, H, 64).transpose(1, 2) for t in qkv.split(D, dim=-1))
    sc = q @ k.transpose(-1, -2)
    if base2:
        sc = (sc - sc.amax(-1, keepdim=True)).exp2()
        p = sc / sc.sum(-1, keepdim=True)
    else:
        p = torch.softmax(sc * scale, dim=-1)
    return p, q, k, v


def _run_short(C, qkv, dout, B, S, H, scale):
    """(out, probs, dqkv) of the short-S kernels in NaN-guarded buffers, plus the guard views"""
    D = H * 64
    ob, out = _nan_buf(B * S * D)
    pb, probs = _nan_buf(B * H * S * _sp(S))
    C.attention_short_fwd(qkv, out.view(B * S, D), probs.view(B * H, S, _sp(S)), B, S, H, 64, scale)
    db = dq = None
    if dout is not None:
        db, dq = _nan_buf(B * S * 3 * D)
        C.attention_short_bwd(qkv, dout, probs.view(B * H, S, _sp(S)), dq.view(B * S, 3 * D), B, S, H, 64, scale)
    torch.cuda.synchronize()
    return (ob, out.view(B * S, D)), (pb, probs.view(B, H, S, _sp(S))), (db, None if dq is None else dq.view(B * S, 3 * D))


def _guard_intact(buf):
    assert torch.isnan(buf[-GUARD:].float()).all(), "a kernel wrote past its output"


def _rne_or_band(got, ref, band=2.0 ** -20):
    """bf16 ``got`` is the nearest-even rounding of float64 ``ref``, or ``ref`` lies within ``band`` (relative) of the
    midpoint between the two neighbours ``got`` and ``rne(ref)``.  Returns (#elements in the band, #taking the other)."""
    rne = ref.to(BF16).double()
    g = got.double()
    other = g != rne
    mid = (g + rne) / 2
    ok = ~other | ((ref - mid).abs() <= band * ref.abs())
    assert ok.all(), "not nearest-even: got {} want {} (ref {})".format(g[~ok][:4].tolist(), rne[~ok][:4].tolist(),
                                                                         ref[~ok][:4].tolist())
    return int(other.sum())


SHAPES = [(17, 2, 3), (65, 40, 3), (65, 48, 6), (101, 20, 3), (127, 5, 6)]   # (S, B, H): B*H 6 .. 288


@pytest.mark.parametrize("S,B,H", SHAPES)
def test_short_attention_forward_exact_family(C, S, B, H):
    g = torch.Generator(device="cpu").manual_seed(S * 1000 + B)
    D = H * 64
    q = torch.zeros(B * S, D)
    k = torch.zeros(B * S, D)
    # four nonzero +-1 entries per row of Q and K: integer scores in [-4, 4]
    for t in (q, k):
        idx = torch.randint(0, 64, (B * S, H, 4), generator=g)
        sgn = torch.randint(0, 2, (B * S, H, 4), generator=g).float() * 2 - 1
        t.view(B * S, H, 64).scatter_(2, idx, sgn)
    v = torch.randint(-4, 5, (B * S, D), generator=g).float()
    qkv = torch.cat([q, k, v], 1).to(BF16).to(DEV).contiguous()
    scale = float(torch.tensor(math.log(2.0), dtype=torch.float32))
    (ob, out), (pb, probs), _ = _run_short(C, qkv, None, B, S, H, scale)
    p, q, k, vv = _ref_attention(qkv, B, S, H, scale, base2=True)
    e = (q @ k.transpose(-1, -2))
    e = (e - e.amax(-1, keepdim=True)).exp2()          # P~: exact powers of two; P~ V and the row sums exact too
    ref_out = ((e @ vv) / e.sum(-1, keepdim=True)).transpose(1, 2).reshape(B * S, D)
    n_out = _rne_or_band(out, ref_out)
    assert (probs[..., S:] == 0).all(), "probs pad columns must be 0"
    n_p = _rne_or_band(probs[..., :S], p)
    print("S={} B={} H={}: out {} / probs {} elements took the other neighbour".format(S, B, H, n_out, n_p))
    _guard_intact(ob)
    _guard_intact(pb)


@pytest.mark.parametrize("S,B,H", SHAPES)
def test_short_attention_bounded_family(C, S, B, H):
    torch.manual_seed(S + 7 * B)
    D = H * 64
    qkv = torch.randn(B * S, 3 * D, device=DEV).to(BF16)
    dout = torch.randn(B * S, D, device=DEV).to(BF16)
    scale = 0.125
    (ob, out), (pb, probs), (db, dqkv) = _run_short(C, qkv, dout, B, S, H, scale)
    p, q, k, v = _ref_attention(qkv, B, S, H, scale)
    do = dout.double().reshape(B, S, H, 64).transpose(1, 2)
    ref_out = p @ v
    win = 2.0 ** -7 * (p @ v.abs()) + 2.0 ** -9 * ref_out.abs()
    got = out.double().reshape(B, S, H, 64).transpose(1, 2)
    assert ((got - ref_out).abs() <= win).all(), float(((got - ref_out).abs() / win).max())
    assert (probs[..., S:] == 0).all()
    assert ((probs[..., :S].double() - p).abs() <= 2.0 ** -8 * p + 1e-30).all()
    # backward in float64 from the same inputs
    dp = do @ v.transpose(-1, -2)
    delta = (p * dp).sum(-1, keepdim=True)
    ds = p * (dp - delta)
    m_ds = p * (dp.abs() + delta.abs())
    refs = {"dq": (scale * ds @ k, scale * m_ds @ k.abs()), "dk": (scale * ds.transpose(-1, -2) @ q,
                                                                   scale * m_ds.transpose(-1, -2) @ q.abs()),
            "dv": (p.transpose(-1, -2) @ do, p.transpose(-1, -2) @ do.abs())}
    worst = {}
    for i, name in enumerate(("dq", "dk", "dv")):
        ref, mag = refs[name]
        g = dqkv[:, i * D:(i + 1) * D].double().reshape(B, S, H, 64).transpose(1, 2)
        win = 2.0 ** -7 * mag + 2.0 ** -9 * ref.abs()
        worst[name] = float(((g - ref).abs() / win).max())
        assert worst[name] <= 1.0, (name, worst[name])
    print("S={} B={} H={}: worst error / window {}".format(S, B, H, worst))
    for b in (ob, pb, db):
        _guard_intact(b)
    (_, out2), (_, probs2), (_, dqkv2) = _run_short(C, qkv, dout, B, S, H, scale)
    assert torch.equal(out2.view(torch.int16), out.view(torch.int16))
    assert torch.equal(probs2.view(torch.int16), probs.view(torch.int16))
    assert torch.equal(dqkv2.view(torch.int16), dqkv.view(torch.int16))


def test_attention_dispatch_and_rejects():
    from baton_b200.ops import nn as bnn
    from baton_b200.ops._ext import launch_counts
    torch.manual_seed(1)
    B, S, H = 4, 65, 3
    qkv = torch.randn(B * S, 3 * H * 64, device=DEV).to(BF16).requires_grad_()
    n0 = launch_counts()
    out = bnn.attention(qkv, B, S, H, 64)
    out.float().sum().backward()
    n = launch_counts() - n0
    assert n.get("attention_short_fwd") == 1 and n.get("attention_short_bwd") == 1, dict(n)
    with pytest.raises(ValueError):
        bnn.attention(qkv.detach(), B, S, H, 64, mask_bias=torch.zeros(B, S, device=DEV))
    x = torch.randn(2 * 65, 3 * 2 * 32, device=DEV).to(BF16)
    with pytest.raises(ValueError):
        bnn.attention(x, 2, 65, 2, 32)


def test_short_attention_matches_sdpa():
    from baton_b200.ops import nn as bnn
    torch.manual_seed(2)
    B, S, H = 16, 65, 6
    qkv = torch.randn(B * S, 3 * H * 64, device=DEV).to(BF16)
    out = bnn.attention(qkv, B, S, H, 64)
    q, k, v = (t.reshape(B, S, H, 64).transpose(1, 2).float() for t in qkv.split(H * 64, dim=-1))
    ref = TF.scaled_dot_product_attention(q, k, v).transpose(1, 2).reshape(B * S, H * 64)
    assert float((out.float() - ref).abs().max() / ref.abs().max()) < 2e-2


# ---------------------------------------------------------------------------------------------------- token kernel
def _dyadic(shape, scale, g, lo=-16, hi=17):
    return torch.randint(lo, hi, shape, generator=g).float() * scale


@pytest.mark.parametrize("B,S,D", [(3, 17, 64), (128, 65, 192), (7, 65, 384), (2, 128, 128)])
def test_token_kernel_exact(C, B, S, D):
    g = torch.Generator().manual_seed(B * S + D)
    z = _dyadic((B, S - 1, D), 1 / 8, g).to(BF16)
    cls, bias, pos = _dyadic((D,), 1 / 64, g), _dyadic((D,), 1 / 64, g), _dyadic((S, D), 1 / 64, g)
    tb, tok = _nan_buf(B * S * D)
    C.vit_tokens_fwd(z.to(DEV), cls.to(DEV), bias.to(DEV), pos.to(DEV), tok.view(B, S, D), B, S, D)
    ref = torch.cat([cls.double().expand(B, 1, D), z.double() + bias.double()], 1) + pos.double()
    assert torch.equal(tok.view(B, S, D).cpu(), ref.to(BF16))
    _guard_intact(tb)
    dtok = _dyadic((B, S, D), 1 / 8, g).to(BF16)
    init = [_dyadic((n,), 1 / 4, g) for n in (D, D, S * D)]
    tgts = [t.to(DEV) for t in init]
    zb, dz = _nan_buf(B * (S - 1) * D)
    C.vit_tokens_bwd(dtok.to(DEV), dz.view(B, S - 1, D), *tgts, B, S, D)
    d = dtok.double()
    assert torch.equal(dz.view(B, S - 1, D).cpu(), dtok[:, 1:])
    _guard_intact(zb)
    want = [init[0].double() + d[:, 0].sum(0), init[1].double() + d[:, 1:].sum((0, 1)),
            init[2].double() + d.sum(0).reshape(-1)]
    for got, w in zip(tgts, want):
        assert torch.equal(got.cpu().double(), w)


def test_token_kernel_deterministic_and_graph(C):
    B, S, D = 128, 65, 192
    torch.manual_seed(3)
    dtok = torch.randn(B, S, D, device=DEV).to(BF16)
    dz = torch.empty(B, S - 1, D, device=DEV, dtype=BF16)

    def run():
        t = [torch.zeros(n, device=DEV) for n in (D, D, S * D)]
        C.vit_tokens_bwd(dtok, dz, *t, B, S, D)
        return t

    a, b = run(), run()
    g = torch.cuda.CUDAGraph()
    t = [torch.zeros(n, device=DEV) for n in (D, D, S * D)]
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        C.vit_tokens_bwd(dtok, dz, *t, B, S, D)     # warm-up outside the capture
        for x in t:
            x.zero_()
        with torch.cuda.graph(g, stream=s):
            C.vit_tokens_bwd(dtok, dz, *t, B, S, D)
    torch.cuda.current_stream().wait_stream(s)
    for x in t:
        x.zero_()
    g.replay()
    torch.cuda.synchronize()
    for x, y, z in zip(a, b, t):
        assert torch.equal(x.view(torch.int32), y.view(torch.int32)) and torch.equal(x.view(torch.int32), z.view(torch.int32))


# ---------------------------------------------------------------------------------------------------- add + LayerNorm
def _ln_ref(s, gamma, beta, eps):
    s = s.double()
    mu = s.mean(-1, keepdim=True)
    var = ((s - mu) ** 2).mean(-1, keepdim=True)
    rs = (var + eps).rsqrt()
    return (s - mu) * rs * gamma.double() + beta.double(), (s - mu) * rs, rs


@pytest.mark.parametrize("rows,D", [(128 * 65, 192), (128 * 65, 384), (33, 64), (1000, 128)])
def test_add_layernorm_against_float64(C, rows, D):
    torch.manual_seed(rows + D)
    x = torch.randn(rows, D, device=DEV).to(BF16)
    r = (torch.randn(rows, D, device=DEV) * 3 + 1).to(BF16)
    gamma = torch.randn(D, device=DEV)
    beta = torch.randn(D, device=DEV)
    eps = 1e-6
    yb, y = _nan_buf(rows * D)
    sb, s = _nan_buf(rows * D)
    mean, rstd = torch.empty(rows, device=DEV), torch.empty(rows, device=DEV)
    C.layernorm_sum_fwd(x, r, y.view(rows, D), s.view(rows, D), gamma, beta, mean, rstd, rows, D, eps)
    s, y = s.view(rows, D), y.view(rows, D)
    assert torch.equal(s, (x.double() + r.double()).to(BF16))
    ref, xhat, rs = _ln_ref(s, gamma, beta, eps)
    ulp = 2.0 ** -8 * ref.abs()
    mag = 2.0 ** -14 * (xhat.abs() * gamma.double().abs() + beta.double().abs())
    assert ((y.double() - ref).abs() <= ulp + mag).all()
    _guard_intact(yb)
    _guard_intact(sb)
    dy = torch.randn(rows, D, device=DEV).to(BF16)
    ds = torch.randn(rows, D, device=DEV).to(BF16)
    g0, b0 = torch.randn(D, device=DEV), torch.randn(D, device=DEV)

    def bwd():
        db_, dsum_ = _nan_buf(rows * D)
        dg, dbt = g0.clone(), b0.clone()
        C.layernorm_sum_bwd(s, dy, ds, dsum_.view(rows, D), gamma, mean, rstd, dg, dbt, rows, D)
        return db_, dsum_.view(rows, D), dg, dbt

    dbuf, dsum, dg, dbt = bwd()
    gw = dy.double() * gamma.double()
    m1, m2 = gw.mean(-1, keepdim=True), (gw * xhat).mean(-1, keepdim=True)
    ref = rs * (gw - m1 - xhat * m2) + ds.double()
    mag = 2.0 ** -14 * (rs * (gw.abs() + m1.abs() + (xhat * m2).abs()) + ds.double().abs())
    err = (dsum.double() - ref).abs()
    assert (err <= 2.0 ** -8 * ref.abs() + mag).all(), float((err / (2.0 ** -8 * ref.abs() + mag)).max())
    _guard_intact(dbuf)
    tg = (dy.double() * xhat).sum(0)
    tb = dy.double().sum(0)
    assert ((dg.double() - g0.double() - tg).abs() <= 2.0 ** -14 * (dy.double() * xhat).abs().sum(0) + 1e-6).all()
    assert ((dbt.double() - b0.double() - tb).abs() <= 2.0 ** -14 * dy.double().abs().sum(0) + 1e-6).all()
    _, dsum2, _, _ = bwd()
    assert torch.equal(dsum2.view(torch.int16), dsum.view(torch.int16))
    # graph replay gives the same dsum bits
    out = torch.empty(rows, D, device=DEV, dtype=BF16)
    dg, dbt = g0.clone(), b0.clone()
    g = torch.cuda.CUDAGraph()
    st = torch.cuda.Stream()
    st.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(st):
        C.layernorm_sum_bwd(s, dy, ds, out, gamma, mean, rstd, dg, dbt, rows, D)
        with torch.cuda.graph(g, stream=st):
            C.layernorm_sum_bwd(s, dy, ds, out, gamma, mean, rstd, dg, dbt, rows, D)
    torch.cuda.current_stream().wait_stream(st)
    out.zero_()
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(out.view(torch.int16), dsum.view(torch.int16))


def test_add_norm_autograd_delivers_skip_gradient():
    from baton_b200.ops import nn as bnn
    from baton_b200.ops._ext import launch_counts
    torch.manual_seed(4)
    ln = bnn.LayerNorm(192, 1e-6).to(DEV)
    x = torch.randn(300, 192, device=DEV).to(BF16).requires_grad_()
    r = torch.randn(300, 192, device=DEV).to(BF16).requires_grad_()
    w = torch.randn(300, 192, device=DEV).to(BF16)
    n0 = launch_counts()
    y, s = ln.add_norm(x, r)
    ((y.float() * w.float()).sum() + (s.float() * 2).sum()).backward()
    n = launch_counts() - n0
    assert n.get("layernorm_sum_fwd") == 1 and n.get("layernorm_sum_bwd") == 1 and not n.get("add"), dict(n)
    xr = (x.detach().double() + r.detach().double()).to(BF16).double().requires_grad_()
    ref = TF.layer_norm(xr, (192,), ln.weight.double(), ln.bias.double(), 1e-6)
    ((ref * w.double()).sum() + (xr * 2).sum()).backward()
    assert torch.equal(x.grad, r.grad)
    assert float((x.grad.double() - xr.grad).abs().max() / xr.grad.abs().max()) < 1e-2


# ---------------------------------------------------------------------------------------------------- erf GELU
def test_gelu_erf_against_float64(C):
    x = torch.linspace(-8, 8, 1 << 16, device=DEV).to(BF16)
    dy = torch.randn(1 << 16, device=DEV).to(BF16)
    y, dx = torch.empty_like(x), torch.empty_like(x)
    C.gelu_erf(x, y)
    C.gelu_erf_bwd(x, dy, dx)
    xd = x.double()
    ref = 0.5 * xd * (1 + torch.erf(xd / math.sqrt(2)))
    dref = dy.double() * (0.5 * (1 + torch.erf(xd / math.sqrt(2))) + xd * torch.exp(-0.5 * xd * xd) / math.sqrt(2 * math.pi))
    assert ((y.double() - ref).abs() <= 2.0 ** -8 * ref.abs() + 2.0 ** -20).all()
    assert ((dx.double() - dref).abs() <= 2.0 ** -8 * dref.abs() + 2.0 ** -20 * dy.double().abs()).all()


# ---------------------------------------------------------------------------------------------------- models
def _tv_vit(m):
    from torchvision.models.vision_transformer import VisionTransformer as TV
    tv = TV(32, 4, len(m.encoder.layers), m.hidden_dim // 64, m.hidden_dim,
            m.encoder.layers[0].mlp[0].out_features, num_classes=10)
    tv.load_state_dict(m.state_dict())
    return tv


def test_vit_tiny_forward_backward_matches_torchvision():
    from baton_b200.models import vit_tiny
    from baton_b200.ops import nn as bnn
    from baton_b200.parallel.arena import ParamArena
    torch.manual_seed(0)
    m = vit_tiny()
    with torch.no_grad():          # a trained-looking head and class token: the fresh ones are zero
        m.heads.head.weight.normal_(std=0.05)
        m.class_token.normal_(std=0.02)
    tv = _tv_vit(m).to(DEV).train()
    ParamArena(m, DEV)
    m.train()
    x = torch.randn(64, 32, 32, 3, device=DEV).to(BF16)
    y = torch.randint(0, 10, (64,), device=DEV)
    logits = m(x)
    ref = tv(x.float().permute(0, 3, 1, 2))
    rel = float((logits - ref).abs().max() / ref.abs().max())
    assert rel < 5e-2, rel
    loss, _ = bnn.cross_entropy(logits, y)
    loss.backward()
    TF.cross_entropy(ref, y).backward()
    params = dict(tv.named_parameters())
    cos = {k: float(TF.cosine_similarity(p.grad.float().flatten(), params[k].grad.flatten(), dim=0))
           for k, p in m.named_parameters()}
    worst = min(cos, key=cos.get)
    print("logits rel {:.4f}; grad cosine vs fp32 mean {:.4f} min {:.4f} ({})".format(
        rel, sum(cos.values()) / len(cos), cos[worst], worst))
    assert sum(cos.values()) / len(cos) > 0.97 and cos[worst] > 0.85, (worst, cos[worst])


def _data(n, seed=0):
    from baton_b200.data import dirichlet_label_shards, image_shard
    spec = dirichlet_label_shards(1, 10, n, 0.5, seed)[0]
    X, y = image_shard(spec, seed=seed, dtype=BF16)
    return X.to(DEV), y.to(DEV)


@pytest.mark.parametrize("use_graph", [True, False])
def test_engine_rounds(use_graph):
    from baton_b200.models import VisionTransformer
    from baton_b200.parallel.engine import FederatedEngine
    torch.manual_seed(0)
    X, y = _data(512)
    m = VisionTransformer(32, 4, 4, 3, 192, 768, 10)
    eng = FederatedEngine(m, DEV, backend="fused", lr=1e-3, batch_size=128, use_graph=use_graph, optimizer="adamw",
                          wire_dtype="fp32")
    hist = []
    for _ in range(4):
        hist += eng.run_round((X, y), n_epoch=1).loss_history
    eng.sync()
    torch.cuda.synchronize()
    print("losses", hist)
    assert all(h == h for h in hist) and hist[-1] < hist[0], hist
    res = eng.evaluate(_data(300, seed=1), batch_size=128)
    assert 0.0 <= res.accuracy <= 1.0 and res.loss == res.loss


def test_engine_round_with_the_deit_recipe():
    from baton_b200.models import VisionTransformer
    from baton_b200.parallel.engine import FederatedEngine
    torch.manual_seed(0)
    X, y = _data(512)
    m = VisionTransformer(32, 4, 2, 3, 192, 768, 10)
    eng = FederatedEngine(m, DEV, backend="fused", lr=1e-3, batch_size=128, optimizer="adamw", wire_dtype="fp32",
                          augment="crop_flip", mix="mixup_cutmix", label_smoothing=0.1, max_grad_norm=1.0)
    hist = []
    for _ in range(2):
        hist += eng.run_round((X, y), n_epoch=1).loss_history
    eng.sync()
    torch.cuda.synchronize()
    assert all(h == h for h in hist), hist
    assert torch.isfinite(eng.arena.theta[: eng.arena.n_param]).all()
