"""Random-crop / horizontal-flip augmentation, CPU tier: the host reference against an independent per-sample
construction, the statistics of the draws, the batches the CPU trainers feed a model, the engine's per-client and
per-round streams, and the configuration and shard checks."""
import argparse

import numpy as np
import pytest
import torch
from torch import nn

from baton_b200.config import FederationConfig
from baton_b200.data.augment import (AugmentConfig, augment_draws, augment_key, check_augment, check_shard,
                                     gather_augment_reference)
from baton_b200.models import FederatedModule, MLP2
from baton_b200.parallel.arena import ParamArena
from baton_b200.parallel.engine import FederatedEngine
from baton_b200.train import PortableLocalSGD, run_local_sgd

KINDS = ["crop", "flip", "crop_flip"]


def _independent(X, idx, key, stream, epoch, padding, crop, flip, s0=0):
    """Per sample: torch.nn.functional.pad, a slice and torch.flip, from the same draws."""
    oy, ox, fl = augment_draws(key, stream, epoch, np.arange(s0, s0 + len(idx)), padding, flip, crop)
    p = padding if crop else 0
    H, W = X.shape[1], X.shape[2]
    out = []
    for j, i in enumerate(idx.tolist()):
        img = X[i].permute(2, 0, 1)                                     # CHW for pad
        img = torch.nn.functional.pad(img, (p, p, p, p))
        img = img[:, oy[j]: oy[j] + H, ox[j]: ox[j] + W]
        if fl[j]:
            img = torch.flip(img, dims=[2])
        out.append(img.permute(1, 2, 0))
    return torch.stack(out)


@pytest.mark.parametrize("shape", [(32, 32, 3), (28, 28, 1), (17, 9, 5)])
@pytest.mark.parametrize("padding", [1, 4, 8])
@pytest.mark.parametrize("kind", KINDS)
def test_reference_equals_pad_slice_flip(shape, padding, kind):
    cfg = check_augment(kind, padding)
    g = torch.Generator().manual_seed(3)
    X = torch.randn((12,) + shape, generator=g)
    idx = torch.tensor([3, 0, 11, 3, 7, 5, 5, 1, 9])
    key, stream = augment_key(5), (2 << 32) | 7
    for epoch, s0 in ((0, 0), (3, 40)):
        got = gather_augment_reference(X, idx, key, stream, epoch, cfg.padding, cfg.crop, cfg.flip, s0=s0)
        want = _independent(X, idx, key, stream, epoch, cfg.padding, cfg.crop, cfg.flip, s0=s0)
        assert torch.equal(got, want)


def test_draws_are_a_pure_function_covering_every_offset_with_fair_flips():
    from scipy import stats
    p, n = 4, 100_000
    pos = np.arange(n)
    a = augment_draws(11, 3, 2, pos, p, True)
    b = augment_draws(11, 3, 2, pos[::-1].copy(), p, True)
    for u, v in zip(a, b):
        assert np.array_equal(u, v[::-1])             # per position, whatever the order it is asked in
    oy, ox, fl = a
    for o in (oy, ox):
        counts = np.bincount(o, minlength=2 * p + 1)
        assert counts.size == 2 * p + 1 and counts.min() > 0
        assert stats.chisquare(counts).pvalue > 1e-4
    assert abs(fl.mean() - 0.5) < 0.01
    # any change of key, stream or epoch gives other draws
    for other in (augment_draws(12, 3, 2, pos[:64], p, True), augment_draws(11, 4, 2, pos[:64], p, True),
                  augment_draws(11, 3, 3, pos[:64], p, True), augment_draws(11, 3 + (1 << 32), 2, pos[:64], p, True)):
        assert not all(np.array_equal(u[:64], v) for u, v in zip(a, other))
    # kinds without crop or flip draw zeros there
    oy0, ox0, _ = augment_draws(11, 3, 2, pos[:64], p, True, crop=False)
    assert not oy0.any() and not ox0.any()
    assert not augment_draws(11, 3, 2, pos[:64], p, False)[2].any()


class Probe(FederatedModule):
    """Records every input batch it is given, in order, into ``rec`` (a device cursor, so captured graphs record on
    replay too)."""
    loss_kind = "mse"

    def __init__(self, shape):
        super().__init__()
        self.lin = nn.Linear(int(np.prod(shape)), 1)

    def start(self, cap, shape, dtype, device):
        self.rec = torch.zeros((cap,) + tuple(shape), dtype=dtype, device=device)
        self.cursor = torch.zeros((), dtype=torch.int64, device=device)
        self.ar = torch.arange(cap, device=device)

    def recorded(self):
        return self.rec[: int(self.cursor)].cpu().clone()

    def forward(self, x):
        b = x.shape[0]
        with torch.no_grad():
            self.rec.index_copy_(0, self.cursor + self.ar[:b], x.detach())
            self.cursor += b
        return self.lin(x.float().flatten(1))


def _fixed_perm(monkeypatch, perms):
    """Every torch.randperm(n) returns perms[n] (on the device asked for)."""
    real = torch.randperm

    def fake(n, *a, device=None, generator=None, **k):
        return perms[n].to(device) if n in perms else real(n, *a, device=device, generator=generator, **k)
    monkeypatch.setattr(torch, "randperm", fake)


def _data(n, shape, seed=0):
    g = torch.Generator().manual_seed(seed)
    return torch.randn((n,) + shape, generator=g), torch.randn(n, generator=g)


def _expect(X, perm, key, stream, n_epoch, cfg):
    return torch.cat([gather_augment_reference(X, perm, key, stream, e, cfg.padding, cfg.crop, cfg.flip)
                      for e in range(n_epoch)])


@pytest.mark.parametrize("trainer", ["run_local_sgd", "portable"])
def test_cpu_trainers_feed_the_reference_batches(monkeypatch, trainer):
    shape, n, bs, n_epoch = (8, 6, 3), 22, 8, 2                 # a ragged last batch of 6
    X, y = _data(n, shape)
    perm = torch.randperm(n, generator=torch.Generator().manual_seed(1))
    _fixed_perm(monkeypatch, {n: perm})
    cfg = AugmentConfig("crop_flip", 2)
    m = Probe(shape)
    m.start(n * n_epoch, shape, X.dtype, "cpu")
    if trainer == "portable":
        tr = PortableLocalSGD(m, ParamArena(m, "cpu"), loss="mse")
        run = lambda **kw: tr.run(X, y, n_epoch=n_epoch, lr=0.01, batch_size=bs, **kw)   # noqa: E731
    else:
        run = lambda **kw: run_local_sgd(m, X, y, n_epoch=n_epoch, lr=0.01, batch_size=bs, loss="mse", **kw)  # noqa
    recs = []
    for _ in range(3):
        m.cursor.zero_()
        run(augment="crop_flip", augment_padding=2, augment_seed=None if len(recs) < 2 else 99)
        recs.append(m.recorded())
    key0 = (tr._aug_streams if trainer == "portable" else m._augment_streams).key
    assert torch.equal(recs[0], _expect(X, perm, key0, 0, n_epoch, cfg))          # run counter 0, then 1
    assert torch.equal(recs[1], _expect(X, perm, key0, 1, n_epoch, cfg))
    assert torch.equal(recs[2], _expect(X, perm, augment_key(99), 2, n_epoch, cfg))
    assert not torch.equal(recs[0][:n], recs[0][n:]), "consecutive epochs must draw afresh"
    assert not torch.equal(recs[0], recs[1]), "a second run must draw afresh"
    # an explicit seed and stream reproduce
    m.cursor.zero_()
    run(augment="crop_flip", augment_padding=2, augment_seed=99, augment_stream=2)
    assert torch.equal(m.recorded(), recs[2])
    # no augmentation: the raw samples
    m.cursor.zero_()
    run()
    assert torch.equal(m.recorded(), X[perm].repeat(n_epoch, 1, 1, 1))


def test_world1_engine_draws_one_stream_per_client_and_round(monkeypatch):
    shape, n_clients = (6, 6, 2), 3
    sizes = {c: 10 + 2 * c for c in range(n_clients)}
    data = {c: _data(sizes[c], shape, seed=c) for c in range(n_clients)}
    perms = {n: torch.arange(n).flip(0) for n in sizes.values()}
    _fixed_perm(monkeypatch, perms)
    m = Probe(shape)
    eng = FederatedEngine(m, "cpu", backend="nccl", loss="mse", lr=0.01, batch_size=4, logical_clients=n_clients,
                          seed=17, augment="crop_flip", augment_padding=2)
    cfg, key = AugmentConfig("crop_flip", 2), augment_key(17)
    m.start(sum(sizes.values()), shape, torch.float32, "cpu")
    seen = {}
    for r in range(2):
        m.cursor.zero_()
        res = eng.run_round(lambda cid: data[cid], n_epoch=1)
        rec, off = m.recorded(), 0
        for cid in res.participants:
            n = sizes[cid]
            X = data[cid][0]
            assert torch.equal(rec[off: off + n], _expect(X, perms[n], key, (r << 32) | cid, 1, cfg)), (r, cid)
            seen[r, cid] = augment_draws(key, (r << 32) | cid, 0, np.arange(n), 2, True)
            off += n
    draws = [np.concatenate(v) for v in seen.values()]
    assert all(not np.array_equal(a[:30], b[:30]) for i, a in enumerate(draws) for b in draws[i + 1:])


def test_config_carries_augmentation_only_when_on():
    base = FederationConfig().train_kwargs()
    assert "augment" not in base and "augment_padding" not in base
    kw = FederationConfig(augment="crop_flip", augment_padding=2).train_kwargs()
    assert kw == dict(base, augment="crop_flip", augment_padding=2)
    parser = argparse.ArgumentParser()
    FederationConfig.add_arguments(parser)
    cfg = FederationConfig.from_args(parser.parse_args(["--augment", "flip", "--augment-padding", "3"]))
    assert (cfg.augment, cfg.augment_padding) == ("flip", 3)
    assert cfg.train_kwargs()["augment"] == "flip"


@pytest.mark.parametrize("kind,padding", [("rotate", 4), ("crop", 0), ("crop_flip", -1), ("crop", 2.5)])
def test_bad_configs_raise(kind, padding):
    with pytest.raises(ValueError):
        check_augment(kind, padding)
    with pytest.raises(ValueError):
        FederationConfig(augment=kind, augment_padding=padding)
    with pytest.raises(ValueError):
        FederatedEngine(MLP2(10, 16, 1), "cpu", backend="nccl", loss="mse", augment=kind, augment_padding=padding)


def test_flip_ignores_padding_and_none_is_off():
    assert check_augment("flip", 0) == AugmentConfig("flip", 0)
    assert check_augment(None) is None and check_augment("none") is None


@pytest.mark.parametrize("X", [torch.zeros(4, 16, dtype=torch.int64), torch.zeros(4, 10), torch.zeros(4, 8, 8),
                               torch.zeros(4, 8, 8, 3, dtype=torch.int64), torch.zeros(4, 4, 8, 3),
                               torch.zeros(4, 8, 4, 3)],
                         ids=["tokens", "2d", "3d", "int-images", "short", "narrow"])
def test_shards_that_cannot_be_augmented_raise(X):
    with pytest.raises(ValueError):
        check_shard(AugmentConfig("crop", 4), X)
    m = MLP2(10, 16, 1)
    y = torch.zeros(X.shape[0])
    with pytest.raises(ValueError):
        run_local_sgd(m, X, y, n_epoch=1, augment="crop", augment_padding=4)
    with pytest.raises(ValueError):
        PortableLocalSGD(m, ParamArena(m, "cpu"), loss="mse").run(X, y, augment="crop", augment_padding=4)
