"""Gradient-norm clipping, CPU tier: validation at every entry point, the portable trainers against a hand-written torch
loop (clip_grad_norm_ after backward, then the FedProx / SCAFFOLD terms, then the step), an engine round with
last_grad_norms(), the configuration field, and the host form of the device kernel's coefficient against torch."""
import numpy as np
import pytest
import torch

from baton_b200.config import FederationConfig
from baton_b200.models import MLP2
from baton_b200.parallel.engine import FederatedEngine
from baton_b200.train import check_max_grad_norm, clip_coefficient, run_local_sgd

from mp_scaffold_gloo import shard  # noqa: E402

BAD = [-1.0, float("inf"), float("nan"), "x", None]


@pytest.mark.parametrize("bad", BAD, ids=["negative", "inf", "nan", "string", "none"])
def test_every_entry_point_rejects_a_bad_threshold(bad):
    X, y = shard(0, 16)
    with pytest.raises(ValueError):
        check_max_grad_norm(bad)
    with pytest.raises(ValueError):
        run_local_sgd(MLP2(10, 16, 1), X, y, n_epoch=1, max_grad_norm=bad)
    with pytest.raises(ValueError):
        FederatedEngine(MLP2(10, 16, 1), "cpu", backend="nccl", loss="mse", max_grad_norm=bad)
    eng = FederatedEngine(MLP2(10, 16, 1), "cpu", backend="nccl", loss="mse")
    with pytest.raises(ValueError):
        eng.trainer.run(X, y, max_grad_norm=bad)
    with pytest.raises(ValueError):
        eng.model.local_train(X, y, n_epoch=1, max_grad_norm=bad)
    with pytest.raises(ValueError):
        FederationConfig(max_grad_norm=bad)


def test_threshold_accepts_zero_and_positive_numbers():
    assert check_max_grad_norm(0) == 0.0 and check_max_grad_norm("1.5") == 1.5


def _by_hand(model, X, y, n_epoch, batch, lr, C, opt_kind, momentum=0.0, wd=0.0, mu=0.0, corr=None):
    """The torch loop the trainers must reproduce: clip right after backward, then the algorithm terms, then the step."""
    params = list(model.parameters())
    anchors = [p.detach().clone() for p in params]
    if opt_kind == "adamw":
        opt = torch.optim.AdamW(params, lr=lr, weight_decay=wd)
    else:
        opt = torch.optim.SGD(params, lr=lr, momentum=momentum, weight_decay=wd)
    perm = torch.randperm(X.shape[0])
    norms = []
    for _ in range(n_epoch):
        norms.append([])
        for idx in torch.split(perm, batch):
            opt.zero_grad(set_to_none=True)
            torch.nn.functional.mse_loss(model(X[idx]), y[idx]).backward()
            norms[-1].append(float(torch.nn.utils.clip_grad_norm_(params, C)))
            with torch.no_grad():
                for p, a in zip(params, anchors):
                    if mu > 0:
                        p.grad.add_(p.detach() - a, alpha=mu)
                if corr is not None:
                    for p, c in zip(params, corr):
                        p.grad.add_(c)
            opt.step()
    return norms


CASES = {
    "sgd_momentum": dict(opt_kind="sgd", momentum=0.9, wd=1e-3),
    "adamw": dict(opt_kind="adamw", wd=0.01),
    "fedprox": dict(opt_kind="sgd", mu=0.5),
    "scaffold": dict(opt_kind="sgd", corr=True),
}


@pytest.mark.parametrize("case", list(CASES))
def test_portable_trainers_equal_a_hand_written_torch_loop(case):
    kw = dict(CASES[case])
    X, y = shard(1, 24)
    C, lr, n_epoch, batch = 5.0, 0.01, 2, 8
    eng = FederatedEngine(MLP2(10, 16, 1), "cpu", backend="nccl", loss="mse", momentum=kw.get("momentum", 0.0))
    ref = MLP2(10, 16, 1)
    ref.load_state_dict(eng.model.state_dict())
    a = eng.arena
    corr_buf = None
    if kw.pop("corr", None):
        corr_buf = torch.randn(a.n_param, generator=torch.Generator().manual_seed(5)) * 0.1
        kw["corr"] = [a._view(corr_buf, a.slots[n]).clone() for n, _ in eng.model.named_parameters()]
    tkw = dict(n_epoch=n_epoch, lr=lr, batch_size=batch, momentum=kw.get("momentum", 0.0),
               weight_decay=kw.get("wd", 0.0), prox_mu=kw.get("mu", 0.0), optimizer=kw["opt_kind"], max_grad_norm=C)
    torch.manual_seed(7)
    eng.trainer.run(X, y, corr=corr_buf, **tkw)
    got = eng.trainer.last_grad_norms()
    torch.manual_seed(7)
    want = _by_hand(ref, X, y, n_epoch, batch, lr, C, **kw)
    for (n, p), q in zip(eng.model.named_parameters(), ref.parameters()):
        assert torch.equal(p, q), n
    assert got == want and sum(v > C for row in want for v in row) >= 3, want
    if corr_buf is None:        # run_local_sgd: the same loop (it has no SCAFFOLD term)
        fn = MLP2(10, 16, 1)
        fn.load_state_dict(eng.model.state_dict())
        ref2 = MLP2(10, 16, 1)
        ref2.load_state_dict(fn.state_dict())
        tkw.pop("batch_size")
        torch.manual_seed(3)
        run_local_sgd(fn, X, y, loss="mse", batch_size=batch, **tkw)
        torch.manual_seed(3)
        _by_hand(ref2, X, y, n_epoch, batch, lr, C, **kw)
        for p, q in zip(fn.parameters(), ref2.parameters()):
            assert torch.equal(p, q)


def test_clipping_changes_the_run_and_zero_is_plain_sgd():
    X, y = shard(2, 32)

    def run(C):
        torch.manual_seed(0)
        m = MLP2(10, 16, 1)
        torch.manual_seed(1)
        run_local_sgd(m, X, y, n_epoch=2, lr=0.01, batch_size=8, max_grad_norm=C)
        return torch.cat([p.detach().flatten() for p in m.parameters()])

    def plain():
        torch.manual_seed(0)
        m = MLP2(10, 16, 1)
        torch.manual_seed(1)
        run_local_sgd(m, X, y, n_epoch=2, lr=0.01, batch_size=8)
        return torch.cat([p.detach().flatten() for p in m.parameters()])

    assert torch.equal(run(0.0), plain())
    assert not torch.allclose(run(1.0), plain())


def test_engine_round_reports_grad_norms_per_client_and_step():
    torch.manual_seed(0)
    eng = FederatedEngine(MLP2(10, 16, 1), "cpu", backend="nccl", loss="mse", lr=0.01, batch_size=8,
                          logical_clients=3, seed=1, max_grad_norm=2.0, wire_dtype="fp32")
    assert eng.last_grad_norms() == {}
    eng.run_round(lambda cid: shard(cid, 16 + 8 * cid), n_epoch=2)
    norms = eng.last_grad_norms()
    assert sorted(norms) == [0, 1, 2]
    for cid, rows in norms.items():
        steps = -(-(16 + 8 * cid) // 8)
        assert len(rows) == 2 and all(len(r) == steps for r in rows), (cid, rows)
        assert all(v > 0 and np.isfinite(v) for r in rows for v in r)
    plain = FederatedEngine(MLP2(10, 16, 1), "cpu", backend="nccl", loss="mse", logical_clients=3)
    plain.run_round(lambda cid: shard(cid, 16), n_epoch=1)
    assert plain.last_grad_norms() == {}


def test_config_round_trips_and_passes_the_threshold_to_workers():
    assert "max_grad_norm" not in FederationConfig().train_kwargs()
    cfg = FederationConfig(max_grad_norm=1.0)
    assert cfg.train_kwargs()["max_grad_norm"] == 1.0
    assert FederationConfig.from_json(cfg.to_json()).max_grad_norm == 1.0
    import argparse
    parser = argparse.ArgumentParser()
    FederationConfig.add_arguments(parser)
    assert FederationConfig.from_args(parser.parse_args(["--max-grad-norm", "0.5"])).max_grad_norm == 0.5


def test_host_coefficient_equals_torch_expression():
    """The device kernel's arithmetic (C rounded to fp32, each operation rounded to fp32) is torch's
    ``clamp(max_norm / (norm + 1e-6), max=1)`` from the fp32 norm, bit for bit, non-finite norms included."""
    g = torch.Generator().manual_seed(0)
    norms = torch.cat([torch.exp(torch.randn(200000, generator=g) * 12.0).float(),
                       torch.tensor([0.0, 1e-45, 1e-38, 3e38, float("inf"), float("nan")])])
    for C in (1.0, 0.1, 3.7, 1e-3, 123.456):
        want = torch.clamp(C / (norms + 1e-6), max=1.0)
        got = torch.from_numpy(clip_coefficient(norms.numpy(), C))
        assert torch.equal(got.view(torch.int32), want.view(torch.int32)), C
