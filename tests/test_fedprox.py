"""FedProx local training, CPU tier: the portable trainers against hand-written FedProx, the SPMD engine on two gloo
ranks, the configuration and command line, and an HTTP round."""
import argparse
import os
import subprocess
import sys

import pytest
import torch

from baton_b200 import data as bdata
from baton_b200.config import FederationConfig
from baton_b200.control import gpu_worker
from baton_b200.demo import LinearTestWorker, main as demo_main, make_app
from baton_b200.models import LinearModel, MLP2
from baton_b200.parallel.arena import ParamArena
from baton_b200.parallel.engine import FederatedEngine
from baton_b200.train import PortableLocalSGD, run_local_sgd
from conftest import run_async
from fedtest import Federation

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _regression(n=40, seed=0):
    g = torch.Generator().manual_seed(seed)
    X = torch.randn(n, 10, generator=g)
    return X, (X @ torch.arange(1.0, 11.0)).unsqueeze(1) + 0.1 * torch.randn(n, 1, generator=g)


def test_run_local_sgd_matches_hand_written_fedprox():
    X, y = _regression()
    lr, mu, bs = 0.01, 0.3, 8
    torch.manual_seed(1)
    model = MLP2(10, 16, 1)
    ref = MLP2(10, 16, 1)
    ref.load_state_dict(model.state_dict())
    hist = run_local_sgd(model, X, y, n_epoch=3, lr=lr, batch_size=bs, loss="mse",
                         generator=torch.Generator().manual_seed(5), prox_mu=mu)
    # hand-written FedProx: the anchor is the model on entry, the term joins the gradient before the plain SGD step
    anchor = [p.detach().clone() for p in ref.parameters()]
    idxs = torch.randperm(X.shape[0], generator=torch.Generator().manual_seed(5))
    for _ in range(3):
        for b in torch.split(idxs, bs):
            ref.zero_grad(set_to_none=True)
            torch.nn.functional.mse_loss(ref(X[b]), y[b]).backward()
            with torch.no_grad():
                for p, a in zip(ref.parameters(), anchor):
                    p.sub_(lr * (p.grad + mu * (p - a)))
    assert len(hist) == 3
    for p, q in zip(model.parameters(), ref.parameters()):
        assert torch.allclose(p, q, rtol=0, atol=1e-6), float((p - q).abs().max())
    assert any(not torch.equal(p, a) for p, a in zip(model.parameters(), anchor))


def test_run_local_sgd_with_zero_prox_mu_is_bit_identical_to_plain_sgd():
    X, y = _regression()
    out = []
    for kw in ({}, {"prox_mu": 0.0}):
        torch.manual_seed(2)
        m = MLP2(10, 16, 1)
        run_local_sgd(m, X, y, n_epoch=2, lr=0.01, batch_size=8, loss="mse", momentum=0.9, weight_decay=1e-3,
                      generator=torch.Generator().manual_seed(3), **kw)
        out.append(torch.cat([p.detach().flatten() for p in m.parameters()]))
    assert torch.equal(out[0], out[1])


def test_prox_mu_must_be_non_negative():
    X, y = _regression()
    with pytest.raises(ValueError):
        run_local_sgd(LinearModel(), X, y, n_epoch=1, prox_mu=-0.1)
    with pytest.raises(ValueError):
        FederatedEngine(LinearModel(), "cpu", backend="nccl", loss="mse", prox_mu=-1.0)
    arena_model = LinearModel()
    tr = PortableLocalSGD(arena_model, ParamArena(arena_model, "cpu"), loss="mse")
    with pytest.raises(ValueError):
        tr.run(X, y, prox_mu=float("nan"))
    with pytest.raises(ValueError):
        FederationConfig(prox_mu=-0.01)


def test_portable_trainer_anchors_on_the_arena_global_copy():
    """One full-batch step of the linear model from theta != global_w: the proximal term pulls toward global_w."""
    torch.manual_seed(0)
    model = LinearModel()
    arena = ParamArena(model, "cpu")
    with torch.no_grad():
        arena.global_w.copy_(arena.theta + torch.linspace(-0.5, 0.5, arena.n))   # the round's global model
    X, y = _regression(16)
    w0, b0 = model.fc1.weight.detach().clone(), model.fc1.bias.detach().clone()
    gw = arena._view(arena.global_w, arena.slots["fc1.weight"]).clone()
    gb = arena._view(arena.global_w, arena.slots["fc1.bias"]).clone()
    lr, mu = 0.05, 0.7
    PortableLocalSGD(model, arena, loss="mse").run(X, y, n_epoch=1, lr=lr, batch_size=16, prox_mu=mu)
    # closed form of one step of mean((X w^T + b - y)^2)
    r = X @ w0.t() + b0 - y                                   # [n, 1]
    gw_loss, gb_loss = 2.0 * (r.t() @ X) / X.shape[0], 2.0 * r.mean(0)
    want_w = w0 - lr * (gw_loss + mu * (w0 - gw))
    want_b = b0 - lr * (gb_loss + mu * (b0 - gb))
    assert torch.allclose(model.fc1.weight, want_w, rtol=0, atol=1e-6)
    assert torch.allclose(model.fc1.bias, want_b, rtol=0, atol=1e-6)
    # anchoring on the weights it was handed instead would give a different step
    assert not torch.allclose(model.fc1.weight, w0 - lr * gw_loss, rtol=0, atol=1e-4)


def test_federated_engine_two_gloo_ranks_fedprox_round():
    port = 29400 + ((os.getpid() + 211) % 500)
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2",
           "--master-addr", "127.0.0.1", "--master-port", str(port), os.path.join(ROOT, "tests", "mp_fedprox_gloo.py")]
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="", OMP_NUM_THREADS="1")
    proc = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=300, cwd=ROOT, env=env)
    tail = "\n".join(proc.stdout.splitlines()[-40:])
    assert proc.returncode == 0 and "RESULT PASS" in proc.stdout, tail


def test_config_json_and_cli_round_trip_prox_mu():
    cfg = FederationConfig(prox_mu=0.01)
    assert FederationConfig.from_json(cfg.to_json()).prox_mu == 0.01
    assert FederationConfig().prox_mu == 0.0
    parser = argparse.ArgumentParser()
    FederationConfig.add_arguments(parser)
    assert FederationConfig.from_args(parser.parse_args(["--prox-mu", "0.1"])).prox_mu == 0.1
    with pytest.raises(SystemExit):
        demo_main(["worker", "127.0.0.1:1", "1", "--prox-mu=-0.5"])


def test_make_app_workers_carry_prox_mu(monkeypatch):
    cfg = FederationConfig(prox_mu=0.05, lr=0.02, batch_size=16)
    app = make_app("worker", "127.0.0.1:1", 1, cfg)
    worker = app["worker"]
    assert worker.train_kwargs == {"lr": 0.02, "batch_size": 16, "prox_mu": 0.05}
    worker._executor.shutdown(wait=False)

    seen = {}

    class FakeSeat:
        def __init__(self, *args, **kwargs):
            seen.update(kwargs)

    monkeypatch.setattr(gpu_worker, "GpuExperimentWorker", FakeSeat)
    monkeypatch.setattr(torch.cuda, "set_device", lambda dev: None)
    monkeypatch.setattr(bdata, "image_shard", lambda *a, **k: (None, None))
    make_app("worker", "127.0.0.1:1", 1, FederationConfig(backend="nccl", prox_mu=0.05, samples_per_client=8))
    assert seen["train_kwargs"]["prox_mu"] == 0.05


@run_async
async def test_http_round_with_prox_mu_stays_closer_to_the_broadcast_model():
    uploads = {}
    for mu in (0.0, 1.0):
        torch.manual_seed(0)
        fed = Federation()
        exp = await fed.start_manager(LinearModel())
        try:
            broadcast = exp.model.fc1.weight.detach().clone()
            w = await fed.add_worker(cls=LinearTestWorker, seed=11, train_kwargs={"lr": 0.02, "prox_mu": mu})
            status, _ = await fed.get("start_round?n_epoch=8")
            assert status == 200
            await fed.wait_round_closed()
            assert exp.update_manager.n_updates == 1
            upload = exp.model.fc1.weight.detach()           # one client: the global model is its upload
            assert torch.equal(upload, w.model.fc1.weight.detach())
            uploads[mu] = float((upload - broadcast).norm())
        finally:
            await fed.close()
    assert 0.0 < uploads[1.0] < uploads[0.0], uploads
