"""GroupNorm on the H100: ``gn_fwd`` / ``gn_bwd`` (csrc/norm.cu) against float64, and GroupNorm ResNets against
torchvision, autograd, eager training and the federation features.

Kernel families:

* **Exact** (flagship shapes, ``M = H*W*C/G`` a power of two).  Each group ``(n, g)`` holds ``m + 2 s`` with an integer
  mean ``m`` and signs ``s = +-1`` split half and half, so the mean is ``m`` and the biased variance exactly 4; with
  ``eps = 0`` rstd must be 0.5.  ``gamma``, ``beta`` are multiples of 1/8, residual and gradient pieces multiples of 1/4.
  Every sum is then exact in fp32 in any order, so ``y``, ``dres`` and ``dz`` must equal the float64 value rounded to
  bf16 (nearest-even), and mean, ``dgamma`` and ``dbeta`` (accumulated into non-zero slots) the float64 value.
* **Bounded** (randn rounded to bf16, means up to 8 standard deviations).  Mean and rstd within ``2^-16`` relative of
  float64; ``y``, ``dz`` within one bf16 ulp plus ``2^-14`` of the magnitude of the terms that cancel; ``dgamma``,
  ``dbeta`` within ``2^-14`` of the sum of the magnitudes of their terms.
"""
import pytest
import torch
from torch.nn import functional as TF

pytestmark = pytest.mark.gpu

BF16 = torch.bfloat16
DEV = torch.device("cuda:0")

# (H, W, C) of every GroupNorm input of ResNet-18 and ResNet-50 on 32x32 images
R18 = [(16, 16, 64), (8, 8, 64), (4, 4, 128), (2, 2, 256), (1, 1, 512)]
R50 = [(16, 16, 64), (8, 8, 64), (8, 8, 256), (8, 8, 128), (4, 4, 128), (4, 4, 512), (4, 4, 256), (2, 2, 256),
       (2, 2, 1024), (2, 2, 512), (1, 1, 512), (1, 1, 2048)]
SHAPES = sorted(set(R18 + R50))
# (residual, relu, two dy pieces): cycled over the shape cases, all eight on the stem shape
VARIANTS = [(r, u, b) for r in (False, True) for u in (False, True) for b in (False, True)]


@pytest.fixture(scope="module")
def F():
    from baton_b200.ops import functional as F
    from baton_b200.ops import load
    load()
    return F


def _cases():
    out = []
    i = 0
    for n in (128, 37):
        for hw_c in SHAPES:
            for g in (1, 2, 32):
                out.append((n, hw_c, g, VARIANTS[i % 8]))
                i += 1
    out += [(128, (16, 16, 64), 2, v) for v in VARIANTS]
    return out


def _ref_fwd(z, res, gamma, beta, G, eps, relu):
    """float64 GroupNorm of NHWC ``z``: -> (y before bf16 rounding, mean [N, G], rstd [N, G], xhat)."""
    n, h, w, c = z.shape
    zg = z.double().reshape(n, h * w, G, c // G)
    mean = zg.mean(dim=(1, 3))
    var = ((zg - mean[:, None, :, None]) ** 2).mean(dim=(1, 3))
    rstd = 1.0 / torch.sqrt(var + eps)
    xhat = ((zg - mean[:, None, :, None]) * rstd[:, None, :, None]).reshape(n, h, w, c)
    y = xhat * gamma.double() + beta.double()
    if res is not None:
        y = y + res.double()
    return (TF.relu(y) if relu else y), mean, rstd, xhat


def _ref_bwd(xhat, y, dy_a, dy_b, gamma, rstd, G, relu):
    """float64 -> (dy', dz, dgamma, dbeta, |terms| of dz, |terms| of dgamma) with the kernel's ReLU mask (y > 0)."""
    n, h, w, c = xhat.shape
    g = dy_a.double() + (dy_b.double() if dy_b is not None else 0.0)
    if relu:
        g = torch.where(y.float() > 0, g, torch.zeros_like(g))
    gg = (g * gamma.double()).reshape(n, h * w, G, c // G)
    xg = xhat.reshape(n, h * w, G, c // G)
    a = gg.mean(dim=(1, 3), keepdim=True)
    b = (gg * xg).mean(dim=(1, 3), keepdim=True)
    r = rstd[:, None, :, None]
    dz = (r * (gg - a - xg * b)).reshape(n, h, w, c)
    mag = (r * (gg.abs() + a.abs() + (xg * b).abs())).reshape(n, h, w, c)
    dgamma = (g * xhat).sum(dim=(0, 1, 2))
    dbeta = g.sum(dim=(0, 1, 2))
    return g, dz, dgamma, dbeta, (g * xhat).abs().sum(dim=(0, 1, 2)), g.abs().sum(dim=(0, 1, 2)), mag


def _exact_inputs(n, h, w, c, G, gen, res_on, dyb_on):
    cg = c // G
    m = h * w * cg
    means = torch.randint(-16, 64, (n, 1, G, 1), generator=gen).double()
    s = torch.ones(n, G, m)
    s[:, :, : m // 2] = -1
    perm = torch.argsort(torch.rand(n, G, m, generator=gen), dim=2)
    signs = torch.gather(s, 2, perm).reshape(n, G, h * w, cg).permute(0, 2, 1, 3)
    z = (means + 2 * signs.double()).reshape(n, h, w, c)
    q = lambda k, d, shape: torch.randint(-k, k + 1, shape, generator=gen).double() / d   # noqa: E731
    gamma, beta = q(8, 8, (c,)), q(8, 8, (c,))
    res = q(8, 4, (n, h, w, c)) if res_on else None
    dy_a = q(8, 4, (n, h, w, c))
    dy_b = q(8, 4, (n, h, w, c)) if dyb_on else None
    prev = q(64, 8, (2, c))                       # non-zero gradient slots to accumulate into
    return z, res, gamma, beta, dy_a, dy_b, prev


def _bounded_inputs(n, h, w, c, G, gen, res_on, dyb_on):
    z = torch.randn(n, h, w, c, generator=gen) + torch.randn(n, 1, 1, c, generator=gen) * 8
    gamma, beta = torch.randn(c, generator=gen), torch.randn(c, generator=gen)
    res = torch.randn(n, h, w, c, generator=gen) if res_on else None
    dy_a = torch.randn(n, h, w, c, generator=gen)
    dy_b = torch.randn(n, h, w, c, generator=gen) if dyb_on else None
    prev = torch.randn(2, c, generator=gen)
    r = lambda t: None if t is None else t.to(BF16).double()   # noqa: E731
    return r(z), r(res), gamma.double(), beta.double(), r(dy_a), r(dy_b), prev.double()


def _run(F, z, res, gamma, beta, dy_a, dy_b, prev, G, eps, relu):
    """Both kernels on the device; NaN-guarded outputs.  -> dict of CPU results."""
    d = lambda t: None if t is None else t.to(DEV)   # noqa: E731
    zb, rb = d(z).to(BF16), None if res is None else d(res).to(BF16)
    gm, bt = d(gamma).float(), d(beta).float()
    n, c = z.shape[0], z.shape[3]
    work = F.gn_work(n, c, G, DEV).fill_(float("nan"))
    y, mean, rstd = F.gn_fwd(zb, rb, gm, bt, G, eps, relu, work)
    dgamma, dbeta = d(prev[0]).float().clone(), d(prev[1]).float().clone()
    dz, dres = F.gn_bwd(zb, y, d(dy_a).to(BF16), None if dy_b is None else d(dy_b).to(BF16), gm, mean, rstd, dgamma,
                        dbeta, G, relu, want_dres=True, work=work)
    torch.cuda.synchronize()
    assert torch.equal(work[:G].view(torch.int32).cpu(), torch.zeros(G, dtype=torch.int32)), "counters not reset"
    return dict(y=y.cpu(), mean=mean.cpu(), rstd=rstd.cpu(), dz=dz.cpu(), dres=dres.cpu(), dgamma=dgamma.cpu(),
                dbeta=dbeta.cpu(), work=work)


def _bf16_ulp(x):
    e = torch.floor(torch.log2(x.abs().clamp_min(2.0 ** -126)))
    return torch.pow(2.0, e - 7)


@pytest.mark.parametrize("n,shape,G,variant", _cases())
def test_exact_on_dyadic_operands(F, n, shape, G, variant):
    h, w, c = shape
    res_on, relu, dyb_on = variant
    gen = torch.Generator().manual_seed(n * 7919 + h * 131 + c + G)
    z, res, gamma, beta, dy_a, dy_b, prev = _exact_inputs(n, h, w, c, G, gen, res_on, dyb_on)
    out = _run(F, z, res, gamma, beta, dy_a, dy_b, prev, G, 0.0, relu)
    y64, mean64, rstd64, xhat = _ref_fwd(z, res, gamma, beta, G, 0.0, relu)
    assert torch.equal(mean64, torch.round(mean64))
    assert torch.equal(out["mean"].double(), mean64)
    assert torch.equal(out["rstd"], torch.full_like(out["rstd"], 0.5))
    assert torch.equal(out["y"], y64.to(BF16))
    g, dz64, dg64, db64, _, _, _ = _ref_bwd(xhat, out["y"], dy_a, dy_b, gamma, rstd64, G, relu)
    assert torch.equal(out["dres"], g.to(BF16))
    assert torch.equal(dz64.float().double(), dz64), "operands not exact in fp32"
    assert torch.equal(out["dz"], dz64.to(BF16))
    assert torch.equal(out["dgamma"].double(), prev[0] + dg64)
    assert torch.equal(out["dbeta"].double(), prev[1] + db64)


LARGE = [(2, (112, 112, 64), 1), (2, (112, 112, 64), 2), (2, (112, 112, 64), 32), (3, (56, 56, 48), 2),
         (5, (7, 7, 2048), 32), (4, (9, 9, 40), 5)]


@pytest.mark.parametrize("n,shape,G,variant", [(n, s, g, VARIANTS[i % 8]) for i, (n, s, g) in enumerate(
    [(128, s, g) for s in R18 for g in (1, 2, 32)] + [(37, s, 2) for s in R50] + LARGE)])
def test_bounded_on_full_mantissa_inputs(F, n, shape, G, variant):
    h, w, c = shape
    res_on, relu, dyb_on = variant
    gen = torch.Generator().manual_seed(n * 31 + h * 17 + c + G)
    z, res, gamma, beta, dy_a, dy_b, prev = _bounded_inputs(n, h, w, c, G, gen, res_on, dyb_on)
    eps = 1e-5
    out = _run(F, z, res, gamma, beta, dy_a, dy_b, prev, G, eps, relu)
    y64, mean64, rstd64, xhat = _ref_fwd(z, res, gamma, beta, G, eps, relu)
    std = 1.0 / rstd64
    assert ((out["mean"].double() - mean64).abs() <= 2.0 ** -16 * (mean64.abs() + std)).all()
    assert ((out["rstd"].double() - rstd64).abs() <= 2.0 ** -16 * rstd64).all()
    mag_y = (xhat * gamma).abs() + beta.abs() + (res.abs() if res is not None else 0)
    err = (out["y"].double() - y64).abs()
    assert (err <= _bf16_ulp(y64) + 2.0 ** -14 * mag_y).all(), float((err / (_bf16_ulp(y64) + 2.0 ** -14 * mag_y)).max())
    g, dz64, dg64, db64, dg_mag, db_mag, dz_mag = _ref_bwd(xhat, out["y"], dy_a, dy_b, gamma, rstd64, G, relu)
    assert torch.equal(out["dres"], g.to(BF16))
    err = (out["dz"].double() - dz64).abs()
    assert (err <= _bf16_ulp(dz64) + 2.0 ** -14 * dz_mag).all()
    assert ((out["dgamma"].double() - prev[0] - dg64).abs() <= 2.0 ** -14 * (dg_mag + prev[0].abs())).all()
    assert ((out["dbeta"].double() - prev[1] - db64).abs() <= 2.0 ** -14 * (db_mag + prev[1].abs())).all()


@pytest.mark.parametrize("n,shape,G", [(128, (16, 16, 64), 2), (128, (1, 1, 512), 32), (2, (112, 112, 64), 2),
                                       (7, (5, 5, 12), 6)])
def test_two_runs_give_identical_bits(F, n, shape, G):
    h, w, c = shape
    gen = torch.Generator().manual_seed(5)
    args = _bounded_inputs(n, h, w, c, G, gen, True, True)
    a = _run(F, *args, G, 1e-5, True)
    b = _run(F, *args, G, 1e-5, True)
    for k in ("y", "mean", "rstd", "dz", "dres", "dgamma", "dbeta"):
        assert torch.equal(a[k], b[k]), k


def test_rejects_groups_not_dividing_channels(F):
    z = torch.zeros(2, 4, 4, 64, device=DEV, dtype=BF16)
    p = torch.ones(64, device=DEV)
    with pytest.raises(RuntimeError):
        F.gn_fwd(z, None, p, p, 3)
    with pytest.raises(RuntimeError):                  # residual of another shape
        F.gn_fwd(z, torch.zeros(2, 4, 4, 32, device=DEV, dtype=BF16), p, p, 2)
    with pytest.raises(RuntimeError):                  # gamma shorter than C
        F.gn_fwd(z, None, p[:32], p, 2)
    y, mean, rstd = F.gn_fwd(z, None, p, p, 2)
    with pytest.raises(RuntimeError):                  # work too small for N x C partials
        F.gn_bwd(z, y, z, None, p, mean, rstd, None, None, 2, work=torch.zeros(8, device=DEV))


# ------------------------------------------------------------------------------------------- models
def _tv_gn(groups=2):
    import torchvision
    return torchvision.models.resnet18(num_classes=10, norm_layer=lambda c: torch.nn.GroupNorm(groups, c))


def _randomize(m):
    from baton_b200.ops import nn as bnn
    g = torch.Generator().manual_seed(7)
    with torch.no_grad():
        for mod in m.modules():
            if isinstance(mod, bnn.GroupNorm):
                mod.weight.copy_(1 + 0.2 * torch.randn(mod.weight.shape, generator=g))
                mod.bias.copy_(0.1 * torch.randn(mod.bias.shape, generator=g))


def _rel(a, b):
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


def test_resnet18_gn_forward_backward_matches_torchvision():
    from baton_b200.models import resnet18
    from baton_b200.ops import nn as bnn
    from baton_b200.parallel.arena import ParamArena
    torch.manual_seed(0)
    m = resnet18(10, norm="group", groups=2)
    _randomize(m)
    tv = _tv_gn()
    tv.load_state_dict(m.state_dict())
    tv = tv.to(DEV).train()
    ParamArena(m, DEV)
    m.build_workspace(DEV)
    m.train()
    x = torch.randn(64, 32, 32, 3, device=DEV)
    y = torch.randint(0, 10, (64,), device=DEV)
    logits = m(x.to(BF16))
    ref = tv(x.to(BF16).float().permute(0, 3, 1, 2))
    assert _rel(logits, ref) < 6e-2, _rel(logits, ref)
    loss, _ = bnn.cross_entropy(logits, y)
    loss.backward()
    TF.cross_entropy(ref, y).backward()
    params = dict(tv.named_parameters())
    fp32 = {k: p.grad.clone() for k, p in params.items()}
    tv.zero_grad()
    with torch.autocast("cuda", dtype=BF16):
        TF.cross_entropy(tv(x.to(BF16).float().permute(0, 3, 1, 2)).float(), y).backward()
    cos = torch.nn.functional.cosine_similarity
    mine = {k: float(cos(p.grad.float().flatten(), fp32[k].flatten(), dim=0)) for k, p in m.named_parameters()}
    stock = {k: float(cos(params[k].grad.float().flatten(), fp32[k].flatten(), dim=0)) for k in mine}
    mean_mine, mean_stock = sum(mine.values()) / len(mine), sum(stock.values()) / len(stock)
    worst = min(mine, key=mine.get)
    print("grad cosine vs fp32: ours mean {:.4f} min {:.4f} ({}), stock autocast mean {:.4f} min {:.4f}".format(
        mean_mine, mine[worst], worst, mean_stock, min(stock.values())))
    assert mean_mine > 0.93 and mean_mine > mean_stock - 0.02, (mean_mine, mean_stock)
    assert mine[worst] > min(stock.values()) - 0.06, (worst, mine[worst], stock[worst])


@pytest.mark.parametrize("arch", ["resnet18", "resnet50"])
def test_explicit_step_matches_autograd(arch):
    from baton_b200 import models
    from baton_b200.ops import nn as bnn
    from baton_b200.ops._ext import launch_counts
    from baton_b200.parallel.arena import ParamArena
    torch.manual_seed(11)
    x = torch.randn(64, 32, 32, 3, device=DEV).to(BF16)
    y = torch.randint(0, 10, (64,), device=DEV)

    def run(explicit):
        torch.manual_seed(3)
        m = getattr(models, arch)(10, norm="group", groups=2)
        _randomize(m)
        arena = ParamArena(m, DEV)
        m.build_workspace(DEV)
        m.train()
        c0 = launch_counts()
        if explicit:
            stats = m.explicit_step(x, y)
        else:
            loss, stats = bnn.cross_entropy(m(x), y)
            loss.backward()
            bnn.WGRAD.join()
        torch.cuda.synchronize()
        counts = launch_counts() - c0
        return stats.clone(), arena.grad.clone(), counts, m, arena
    s1, g1, c1, m, arena = run(True)
    s2, g2, c2, _, _ = run(False)
    n_gn = sum(isinstance(mod, bnn.GroupNorm) for mod in m.modules())
    assert c1["gn_fwd"] == n_gn and c1["gn_bwd"] == n_gn, c1
    assert not any(k.startswith("bn_") for k in c1), c1
    assert abs(float(s1[0]) - float(s2[0])) < 1e-2 * abs(float(s2[0]))
    assert _rel(g1, g2) < 2e-2, _rel(g1, g2)
    for name, slot in arena.slots.items():
        a, b = g1[slot.offset: slot.offset + slot.numel], g2[slot.offset: slot.offset + slot.numel]
        if b.norm() > 0:
            assert float(torch.nn.functional.cosine_similarity(a, b, dim=0)) > 0.99, name


def _trainer(use_graph, seed=0):
    from baton_b200.models import resnet18
    from baton_b200.parallel.arena import ParamArena
    from baton_b200.train import GraphedLocalSGD
    torch.manual_seed(seed)
    m = resnet18(10, norm="group")
    arena = ParamArena(m, DEV, momentum=True)
    m.build_workspace(DEV)
    tr = GraphedLocalSGD(m, arena, loss="ce", use_graph=use_graph)
    m._graphed_trainer = tr
    return m, arena, tr


def _data(n=1024):
    from baton_b200.data import ShardSpec, image_shard
    X, y = image_shard(ShardSpec(0, torch.full((10,), 0.1), n), noise=0.3)
    return X.to(DEV).to(BF16), y.to(DEV)


def test_graphed_and_eager_local_sgd_agree_and_learn():
    X, y = _data()
    out = []
    for use_graph in (True, False):
        m, arena, tr = _trainer(use_graph)
        torch.manual_seed(9)
        hist = m.train(X, y, n_epoch=4, lr=0.05, batch_size=128, momentum=0.9)
        torch.cuda.synchronize()
        out.append((hist, arena.theta[: arena.n_param].clone()))
    (hg, tg), (he, te) = out
    print("graphed losses", hg, "eager losses", he)
    assert hg[-1] < hg[0] * 0.7, hg
    assert _rel(tg, te) < 1e-2, _rel(tg, te)
    assert all(abs(a - b) < 2e-2 * abs(b) for a, b in zip(hg, he)), (hg, he)


def _engine(**kw):
    from baton_b200.models import resnet18
    from baton_b200.parallel.engine import FederatedEngine
    torch.manual_seed(0)
    model = resnet18(10, norm="group")
    if kw.pop("fp8_convs", False):
        model.set_precision("fp8")
    return FederatedEngine(model, DEV, backend="fused", lr=kw.pop("lr", 0.05), batch_size=128, n_ctas=64, **kw)


def test_engine_round_and_evaluate_use_the_group_norm_kernels():
    from baton_b200.ops import nn as bnn
    X, y = _data(512)
    eng = _engine()
    hist = []
    for _ in range(3):
        hist += eng.run_round((X, y), n_epoch=1).loss_history
    eng.sync()
    torch.cuda.synchronize()
    assert all(h == h for h in hist) and hist[-1] < hist[0], hist
    Xe, ye = _data(300)
    res = eng.evaluate((Xe, ye), batch_size=128)
    assert eng.trainer.eval_launches["gn_fwd"] == 20 * 3, eng.trainer.eval_launches
    m = eng.model
    torch.nn.Module.train(m, False)
    with torch.no_grad():
        logits = torch.cat([m(Xe[s: s + 128]).float() for s in range(0, 300, 128)])
    loss = float(TF.cross_entropy(logits, ye))
    acc = float((logits.argmax(1) == ye).float().mean())
    print("held-out loss {:.4f} accuracy {:.4f}".format(res.loss, res.accuracy))
    assert abs(res.loss - loss) < 1e-4 * max(1.0, loss), (res.loss, loss)
    assert abs(res.accuracy - acc) < 1e-9, (res.accuracy, acc)
    assert not any(isinstance(mod, bnn.BatchNorm2d) for mod in m.modules())


@pytest.mark.parametrize("feature", ["adamw", "clip", "fedprox", "dp", "fp8_wire", "fp8_convs"])
def test_engine_round_with_feature(feature):
    X, y = _data(512)
    kw = {"adamw": dict(optimizer="adamw", lr=1e-3, wire_dtype="fp32"), "clip": dict(max_grad_norm=1.0),
          "fedprox": dict(prox_mu=0.01), "dp": dict(dp_clip=5.0, dp_noise_multiplier=0.0, dp_seed=3, wire_dtype="fp32"),
          "fp8_wire": dict(wire_dtype="fp8"), "fp8_convs": dict(fp8_convs=True)}[feature]
    eng = _engine(**kw)
    hist = []
    for _ in range(3):
        hist += eng.run_round((X, y), n_epoch=1).loss_history
    eng.sync()
    torch.cuda.synchronize()
    print(feature, hist)
    assert all(h == h for h in hist) and hist[-1] < hist[0], hist
    sd = eng.model.state_dict()
    assert all(torch.isfinite(v).all() for v in sd.values())
