"""Mixup, CutMix and label smoothing, CPU tier: the per-batch draws of ``mix_table``, the host reference of the mixed
batch, the soft-target loss against torch's cross-entropy, one step of each CPU trainer against a hand-written torch
computation, the engine's per-client streams, and the option checks of the engine, the config and the trainers."""
import argparse
import json
import math

import numpy as np
import pytest
import torch
from torch import nn

from baton_b200.config import FederationConfig
from baton_b200.data.augment import augment_key, gather_augment_reference
from baton_b200.data.mix import (CUTMIX, MIXUP, MixConfig, check_mix, decode_row, mix_batch_reference, mix_table,
                                 soft_cross_entropy, soft_hits)
from baton_b200.models import FederatedModule, MLP2
from baton_b200.parallel.arena import ParamArena
from baton_b200.parallel.engine import FederatedEngine
from baton_b200.train import PortableLocalSGD, run_local_sgd

H, W = 32, 32


def _rows(kind, n=2000, alpha=1.0, key=5, stream=7, epoch=0):
    return [decode_row(r) for r in mix_table(key, stream, epoch, n, MixConfig(kind, alpha, 0.0), H, W)]


# ---------------------------------------------------------------------------------------------------- draws
def test_mix_table_is_deterministic_and_independent_across_streams_and_epochs():
    cfg = MixConfig("mixup_cutmix", 1.0, 0.0)
    a = mix_table(11, 3, 2, 64, cfg, H, W)
    assert np.array_equal(a, mix_table(11, 3, 2, 64, cfg, H, W))
    assert np.array_equal(a[:10], mix_table(11, 3, 2, 10, cfg, H, W)), "row b must not depend on n_batches"
    for other in (mix_table(12, 3, 2, 64, cfg, H, W), mix_table(11, 4, 2, 64, cfg, H, W),
                  mix_table(11, 3, 3, 64, cfg, H, W), mix_table(11, 3 + (1 << 32), 2, 64, cfg, H, W)):
        assert not np.array_equal(a, other)
    assert a.dtype == np.int32 and a.shape == (64, 8)


@pytest.mark.parametrize("hw", [(32, 32), (28, 20), (7, 5)])
def test_cutmix_boxes_lie_inside_and_set_lam(hw):
    h, w = hw
    for r in (decode_row(x) for x in mix_table(1, 2, 0, 500, MixConfig("cutmix", 1.0, 0.0), h, w)):
        assert r.kind == CUTMIX
        assert 0 <= r.y0 <= r.y1 <= h and 0 <= r.x0 <= r.x1 <= w
        want = 1.0 - (r.y1 - r.y0) * (r.x1 - r.x0) / (h * w)
        assert r.lam == np.float32(want) and r.lam1 == np.float32(1.0 - want)


def test_mixup_rows_draw_beta_lambda_with_mean_one_half():
    rows = _rows("mixup", n=4000)
    lam = np.array([r.lam for r in rows])
    assert all(r.kind == MIXUP and (r.y0, r.y1, r.x0, r.x1) == (0, 0, 0, 0) for r in rows)
    assert abs(lam.mean() - 0.5) < 0.02 and lam.min() >= 0.0 and lam.max() <= 1.0
    assert all(r.lam1 == np.float32(1.0 - np.float64(r.lam)) or abs(r.lam + r.lam1 - 1.0) < 1e-6 for r in rows)
    # a small alpha pushes lambda to the ends
    lam_small = np.array([r.lam for r in _rows("mixup", n=4000, alpha=0.2)])
    assert np.mean(np.minimum(lam_small, 1 - lam_small)) < np.mean(np.minimum(lam, 1 - lam))


def test_mixup_cutmix_yields_both_kinds():
    kinds = np.array([r.kind for r in _rows("mixup_cutmix", n=1000)])
    assert 0.4 < (kinds == CUTMIX).mean() < 0.6 and set(kinds.tolist()) == {MIXUP, CUTMIX}


# ---------------------------------------------------------------------------------------------------- reference
def _row(lam, kind=MIXUP, box=(0, 0, 0, 0)):
    w = np.zeros(8, dtype=np.int32)
    w[:2] = np.array([lam, 1.0 - lam], dtype=np.float32).view(np.int32)
    w[2] = kind
    w[3:7] = box
    return torch.from_numpy(w)


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16, torch.float16])
def test_cutmix_copies_the_partners_box_and_keeps_its_own_pixels(dtype):
    g = torch.Generator().manual_seed(0)
    x = torch.randn(5, 12, 10, 3, generator=g).to(dtype)
    y = torch.arange(5)
    out, t = mix_batch_reference(x, y, _row(0.0, CUTMIX, (2, 9, 3, 7)), 0.1)
    inside = torch.zeros(12, 10, dtype=torch.bool)
    inside[2:9, 3:7] = True
    for j in range(5):
        p = (j - 1) % 5
        assert torch.equal(out[j][inside], x[p][inside]) and torch.equal(out[j][~inside], x[j][~inside])
    assert t.b.tolist() == [4, 0, 1, 2, 3] and t.eps == 0.1


def test_mixup_with_lam_one_is_the_identity_and_rounds_each_product():
    x = torch.randn(4, 6, 6, 3).to(torch.bfloat16)
    out, t = mix_batch_reference(x, torch.arange(4), _row(1.0), 0.0)
    assert torch.equal(out, x) and t.lam == 1.0 and t.lam1 == 0.0
    lam = 0.3
    out, _ = mix_batch_reference(x, torch.arange(4), _row(lam), 0.0)
    l32, l132 = np.float32(lam), np.float32(1.0 - lam)
    a, b = x.float().numpy(), x.roll(1, 0).float().numpy()
    want = (a * l32).astype(np.float32) + (b * l132).astype(np.float32)
    assert torch.equal(out, torch.from_numpy(want.astype(np.float32)).to(torch.bfloat16))


def test_partners_roll_within_a_ragged_batch():
    x = torch.arange(3, dtype=torch.float32).reshape(3, 1, 1, 1).expand(3, 4, 4, 1).contiguous()
    out, t = mix_batch_reference(x, torch.tensor([7, 8, 9]), _row(0.0, CUTMIX, (0, 4, 0, 4)), 0.0)
    assert out[:, 0, 0, 0].tolist() == [2.0, 0.0, 1.0] and t.b.tolist() == [9, 7, 8]
    one, t1 = mix_batch_reference(x[:1], torch.tensor([5]), _row(0.25), 0.0)
    assert torch.equal(one, x[:1]) and t1.b.tolist() == [5]


# ---------------------------------------------------------------------------------------------------- loss
def _soft_loss_f64(z, a, b, lam, lam1, eps):
    z = z.double()
    C = z.shape[1]
    q = torch.full_like(z, eps / C)
    q += (1 - eps) * lam * nn.functional.one_hot(a, C).double()
    q += (1 - eps) * lam1 * nn.functional.one_hot(b, C).double()
    return (torch.logsumexp(z, 1) - (q * z).sum(1)).mean(), torch.softmax(z, 1) - q


@pytest.mark.parametrize("eps", [0.0, 0.1, 0.5])
@pytest.mark.parametrize("lam", [1.0, 0.7, 0.0])
def test_soft_cross_entropy_equals_the_explicit_soft_target(eps, lam):
    g = torch.Generator().manual_seed(1)
    z = torch.randn(9, 10, generator=g, dtype=torch.float64, requires_grad=True)
    a = torch.randint(0, 10, (9,), generator=g)
    _, t = mix_batch_reference(torch.zeros(9, 2, 2, 1), a, _row(lam), eps)
    got = soft_cross_entropy(z, t)
    want, grad = _soft_loss_f64(z.detach(), a, a.roll(1, 0), t.lam, t.lam1, eps)
    assert abs(float(got.detach()) - float(want)) < 1e-6
    got.backward()
    assert torch.allclose(z.grad * 9, grad, atol=1e-6)
    if eps == 0.0 and lam == 1.0:
        assert float(got.detach()) == pytest.approx(float(nn.functional.cross_entropy(z.detach().float(), a)), abs=1e-6)


def test_soft_hits_weight_both_labels():
    z = torch.eye(4) * 5                       # argmax = row index
    _, t = mix_batch_reference(torch.zeros(4, 2, 2, 1), torch.tensor([0, 1, 3, 3]), _row(0.75), 0.0)
    # own label hits rows 0, 1, 3; partner labels [3, 0, 1, 3] hit row 3
    assert float(soft_hits(z, t)) == pytest.approx(0.75 * 3 + 0.25 * 1)


def test_cpu_cross_entropy_takes_the_mix_argument():
    from baton_b200.ops import nn as bnn
    z = torch.randn(6, 5)
    y = torch.randint(0, 5, (6,))
    row = _row(0.4)
    loss, stats = bnn.cross_entropy(z, y, mix=(row, 0.2))
    _, t = mix_batch_reference(torch.zeros(6, 1, 1, 1), y, row, 0.2)
    assert float(loss) == pytest.approx(float(soft_cross_entropy(z, t)))
    assert float(stats[1]) == pytest.approx(float(soft_hits(z, t)))
    loss0, _ = bnn.cross_entropy(z, y, mix=(None, 0.0))
    assert float(loss0) == pytest.approx(float(nn.functional.cross_entropy(z, y)))


# ---------------------------------------------------------------------------------------------------- trainers
class Classifier(FederatedModule):
    loss_kind = "ce"

    def __init__(self, shape, classes=10):
        super().__init__()
        self.lin = nn.Linear(int(np.prod(shape)), classes)

    def forward(self, x):
        return self.lin(x.float().flatten(1))


def _fixed_perm(monkeypatch, perms):
    real = torch.randperm

    def fake(n, *a, device=None, generator=None, **k):
        return perms[n].to(device) if n in perms else real(n, *a, device=device, generator=generator, **k)
    monkeypatch.setattr(torch, "randperm", fake)


@pytest.mark.parametrize("kind", ["mixup", "cutmix"])
@pytest.mark.parametrize("trainer", ["run_local_sgd", "portable"])
def test_cpu_trainer_step_equals_hand_written_torch(monkeypatch, trainer, kind):
    shape, n, eps, lr, seed, stream = (8, 8, 3), 12, 0.1, 0.5, 21, 3
    g = torch.Generator().manual_seed(4)
    X, y = torch.randn((n,) + shape, generator=g), torch.randint(0, 10, (n,), generator=g)
    perm = torch.randperm(n, generator=g)
    _fixed_perm(monkeypatch, {n: perm})
    torch.manual_seed(0)
    m = Classifier(shape)
    w0 = {k: v.detach().clone() for k, v in m.named_parameters()}
    kw = dict(n_epoch=1, lr=lr, batch_size=n, augment="crop_flip", augment_padding=2, augment_seed=seed,
              augment_stream=stream, mix=kind, mix_alpha=0.7, label_smoothing=eps)
    if trainer == "portable":
        tr = PortableLocalSGD(m, ParamArena(m, "cpu"), loss="ce")
        tr.run(X, y, **kw)
        acc = tr.last_stats["accuracy"][0]
    else:
        run_local_sgd(m, X, y, loss="ce", **kw)
    # by hand: crop/flip, then the batch rolled by one under row 0 of epoch 0, and the explicit soft target
    key = augment_key(seed)
    xa = gather_augment_reference(X, perm, key, stream, 0, 2, True, True)
    r = decode_row(mix_table(key, stream, 0, 1, MixConfig(kind, 0.7, eps), H=8, W=8)[0])
    partner = xa.roll(1, 0)
    if r.kind == CUTMIX:
        xm = xa.clone()
        xm[:, r.y0:r.y1, r.x0:r.x1] = partner[:, r.y0:r.y1, r.x0:r.x1]
    else:
        xm = (xa * np.float32(r.lam)) + (partner * np.float32(r.lam1))
    lin = nn.Linear(int(np.prod(shape)), 10)
    with torch.no_grad():
        lin.weight.copy_(w0["lin.weight"])
        lin.bias.copy_(w0["lin.bias"])
    z = lin(xm.flatten(1))
    ya = y[perm]
    C = 10
    q = eps / C + (1 - eps) * (r.lam * nn.functional.one_hot(ya, C) + r.lam1 * nn.functional.one_hot(ya.roll(1, 0), C))
    loss = (torch.logsumexp(z, 1) - (q * z).sum(1)).mean()
    loss.backward()
    with torch.no_grad():
        assert torch.allclose(m.lin.weight, w0["lin.weight"] - lr * lin.weight.grad, atol=1e-5)
        assert torch.allclose(m.lin.bias, w0["lin.bias"] - lr * lin.bias.grad, atol=1e-5)
    if trainer == "portable":
        am = z.argmax(1)
        want = (r.lam * (am == ya).sum() + r.lam1 * (am == ya.roll(1, 0)).sum()) / n
        assert acc == pytest.approx(float(want), abs=1e-6)


def test_label_smoothing_alone_needs_no_image_shard():
    m = MLP2(6, 8, 3)
    m.loss_kind = "ce"
    X, y = torch.randn(10, 6), torch.randint(0, 3, (10,))
    tr = PortableLocalSGD(m, ParamArena(m, "cpu"), loss="ce")
    losses = tr.run(X, y, n_epoch=2, lr=0.1, batch_size=4, label_smoothing=0.2)
    assert all(math.isfinite(v) for v in losses)


class Probe(Classifier):
    """Records every input batch it is given, in order."""

    def start(self):
        self.rec = []

    def forward(self, x):
        self.rec.append(x.detach().clone())
        return super().forward(x)


def test_world1_engine_mixes_with_one_stream_per_client_and_round(monkeypatch):
    shape, n_clients, bs = (6, 6, 2), 3, 4
    sizes = {c: 10 + 2 * c for c in range(n_clients)}
    g = torch.Generator().manual_seed(9)
    data = {c: (torch.randn((sizes[c],) + shape, generator=g), torch.randint(0, 10, (sizes[c],), generator=g))
            for c in range(n_clients)}
    perms = {n: torch.arange(n).flip(0) for n in sizes.values()}
    _fixed_perm(monkeypatch, perms)
    m = Probe(shape)
    eng = FederatedEngine(m, "cpu", backend="nccl", loss="ce", lr=0.01, batch_size=bs, logical_clients=n_clients,
                          seed=17, mix="mixup_cutmix", label_smoothing=0.1)
    key, cfg = augment_key(17), MixConfig("mixup_cutmix", 1.0, 0.1)
    for r in range(2):
        m.start()
        res = eng.run_round(lambda cid: data[cid], n_epoch=1)
        assert all(math.isfinite(v) for v in res.loss_history)
        got = iter(m.rec)
        for cid in res.participants:
            X, y = data[cid]
            n = sizes[cid]
            rows = mix_table(key, (r << 32) | cid, 0, (n + bs - 1) // bs, cfg, 6, 6)
            for b, idx in enumerate(torch.split(perms[n], bs)):
                want, _ = mix_batch_reference(X[idx], y[idx], rows[b], 0.1)
                assert torch.equal(next(got), want), (r, cid, b)


# ---------------------------------------------------------------------------------------------------- options
def test_config_carries_mixing_and_smoothing_only_when_on():
    base = FederationConfig().train_kwargs()
    assert not {"mix", "mix_alpha", "label_smoothing"} & set(base)
    kw = FederationConfig(mix="cutmix", mix_alpha=0.4, label_smoothing=0.1).train_kwargs()
    assert kw == dict(base, mix="cutmix", mix_alpha=0.4, label_smoothing=0.1)
    assert FederationConfig(label_smoothing=0.2).train_kwargs() == dict(base, label_smoothing=0.2)
    cfg = FederationConfig(mix="mixup_cutmix", mix_alpha=0.2, label_smoothing=0.05)
    back = FederationConfig.from_json(cfg.to_json())
    assert (back.mix, back.mix_alpha, back.label_smoothing) == ("mixup_cutmix", 0.2, 0.05)
    assert json.loads(cfg.to_json())["mix"] == "mixup_cutmix"
    parser = argparse.ArgumentParser()
    FederationConfig.add_arguments(parser)
    ns = parser.parse_args(["--mix", "mixup", "--mix-alpha", "0.3", "--label-smoothing", "0.1"])
    cfg = FederationConfig.from_args(ns)
    assert (cfg.mix, cfg.mix_alpha, cfg.label_smoothing) == ("mixup", 0.3, 0.1)
    assert cfg.train_kwargs()["mix"] == "mixup"


def test_none_and_zero_are_off():
    assert check_mix(None) is None and check_mix("none", 1.0, 0.0) is None
    assert check_mix(None, 1.0, 0.1) == MixConfig(None, 1.0, 0.1)
    assert check_mix("cutmix", 2, 0) == MixConfig("cutmix", 2.0, 0.0)


BAD = [dict(mix="blend"), dict(mix="mixup", mix_alpha=0.0), dict(mix="mixup", mix_alpha=-1.0),
       dict(mix="mixup", mix_alpha=float("inf")), dict(mix="mixup", mix_alpha=float("nan")),
       dict(label_smoothing=1.0), dict(label_smoothing=-0.1), dict(mix="cutmix", label_smoothing=float("nan"))]


@pytest.mark.parametrize("opts", BAD, ids=[str(b) for b in BAD])
def test_bad_options_raise(opts):
    with pytest.raises(ValueError):
        check_mix(opts.get("mix"), opts.get("mix_alpha", 1.0), opts.get("label_smoothing", 0.0))
    with pytest.raises(ValueError):
        FederationConfig(**opts)
    with pytest.raises(ValueError):
        FederatedEngine(Classifier((4, 4, 1)), "cpu", backend="nccl", **opts)
    m = Classifier((4, 4, 1))
    X, y = torch.randn(4, 4, 4, 1), torch.randint(0, 10, (4,))
    with pytest.raises(ValueError):
        PortableLocalSGD(m, ParamArena(m, "cpu"), loss="ce").run(X, y, **opts)
    with pytest.raises(ValueError):
        run_local_sgd(m, X, y, n_epoch=1, loss="ce", **opts)


@pytest.mark.parametrize("opts", [dict(mix="mixup"), dict(label_smoothing=0.1)])
def test_mse_and_callable_losses_raise(opts):
    with pytest.raises(ValueError):
        FederatedEngine(MLP2(10, 16, 1), "cpu", backend="nccl", loss="mse", **opts)
    m = MLP2(16, 8, 1)
    X, y = torch.randn(4, 4, 4, 1), torch.randn(4)
    with pytest.raises(ValueError):
        PortableLocalSGD(m, ParamArena(m, "cpu"), loss="mse").run(X, y, **opts)
    with pytest.raises(ValueError):
        run_local_sgd(m, X, y, n_epoch=1, loss="mse", **opts)
    with pytest.raises(ValueError):
        run_local_sgd(m, X, y, n_epoch=1, loss=nn.functional.mse_loss, **opts)


@pytest.mark.parametrize("X", [torch.zeros(4, 16, dtype=torch.int64), torch.zeros(4, 10), torch.zeros(4, 8, 8),
                               torch.zeros(4, 8, 8, 3, dtype=torch.int64)],
                         ids=["tokens", "2d", "3d", "int-images"])
def test_mixing_shards_that_are_not_images_raises(X):
    m = Classifier((10,))
    y = torch.zeros(X.shape[0], dtype=torch.int64)
    with pytest.raises(ValueError):
        PortableLocalSGD(m, ParamArena(m, "cpu"), loss="ce").run(X, y, mix="cutmix")
    with pytest.raises(ValueError):
        run_local_sgd(m, X, y, n_epoch=1, loss="ce", mix="mixup")
