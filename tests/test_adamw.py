"""Local AdamW, CPU tier: the rejections of the engine, the trainers and the configuration, the per-step coefficient
table against torch.optim.AdamW, the SPMD engine with logical clients against a hand-written "fresh AdamW per client
per round, then the FedAvg mean", and the same across two gloo ranks."""
import math
import os
import subprocess
import sys

import pytest
import torch

from baton_b200.config import FederationConfig
from baton_b200.models import MLP2
from baton_b200.ops import functional as F
from baton_b200.parallel.engine import FederatedEngine
from baton_b200.train import run_local_sgd

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

from mp_adamw_gloo import EPOCHS, global_error, make_engine  # noqa: E402
from mp_scaffold_gloo import shard  # noqa: E402


@pytest.mark.parametrize("kw", [{"momentum": 0.9}, {"prox_mu": 0.01}, {"scaffold": True}, {"betas": (1.0, 0.999)},
                                {"betas": (0.9, -0.1)}, {"eps": 0.0}, {"optimizer": "adam"}],
                         ids=["momentum", "fedprox", "scaffold", "beta1", "beta2", "eps", "unknown"])
def test_engine_rejects_unsupported_combinations(kw):
    kw = dict({"optimizer": "adamw"}, **kw)
    with pytest.raises(ValueError):
        FederatedEngine(MLP2(10, 16, 1), "cpu", backend="nccl", loss="mse", **kw)


def test_trainers_reject_sgd_terms():
    X, y = shard(0, 16)
    with pytest.raises(ValueError):
        run_local_sgd(MLP2(10, 16, 1), X, y, n_epoch=1, optimizer="adamw", momentum=0.9)
    eng = FederatedEngine(MLP2(10, 16, 1), "cpu", backend="nccl", loss="mse")
    with pytest.raises(ValueError):
        eng.trainer.run(X, y, optimizer="adamw", prox_mu=0.1)
    with pytest.raises(ValueError):
        eng.trainer.run(X, y, optimizer="adamw", corr=torch.zeros(eng.arena.n_param))


@pytest.mark.parametrize("kw", [{"optimizer": "lamb"}, {"adam_beta1": 1.0}, {"adam_beta2": -0.5}, {"adam_eps": 0.0},
                                {"optimizer": "adamw", "momentum": 0.9}, {"optimizer": "adamw", "prox_mu": 0.1}])
def test_config_rejects_bad_adamw_values(kw):
    with pytest.raises(ValueError):
        FederationConfig(**kw)


def test_config_passes_adamw_to_workers():
    assert "optimizer" not in FederationConfig().train_kwargs()
    kw = FederationConfig(optimizer="adamw", adam_beta1=0.8, adam_beta2=0.95, adam_eps=1e-6).train_kwargs()
    assert kw["optimizer"] == "adamw" and kw["betas"] == (0.8, 0.95) and kw["eps"] == 1e-6


def test_cli_reports_bad_adamw_values_as_usage_errors():
    proc = subprocess.run([sys.executable, "-m", "baton_b200.demo", "worker", "h:1", "1", "--adam-beta2", "1.5"],
                          stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True, timeout=120, cwd=ROOT,
                          env=dict(os.environ, CUDA_VISIBLE_DEVICES=""))
    assert proc.returncode == 2 and "beta2" in proc.stderr, proc.stderr[-2000:]


@pytest.mark.parametrize("n, batch, n_epoch", [(12, 4, 3), (10, 4, 3), (7, 7, 2)], ids=["even", "ragged", "full"])
def test_step_table_matches_torch_adamw(n, batch, n_epoch):
    """Row ``e * steps + s`` (the row step ``s`` of epoch ``e`` reads, the ragged step being the last of its epoch)
    holds the coefficients torch.optim.AdamW uses at that step, and replaying a scalar run through the rows tracks
    torch's parameter."""
    lr, betas, eps, wd = 0.03, (0.85, 0.98), 1e-7, 0.1
    steps = -(-n // batch)
    rows = F.adamw_rows(lr, betas, eps, wd, 1, n_epoch * steps)
    assert rows.shape == (n_epoch * steps, F.ADAMW_ROW) and rows.dtype == torch.float32
    p = torch.nn.Parameter(torch.tensor([0.7], dtype=torch.float64))
    opt = torch.optim.AdamW([p], lr=lr, betas=betas, eps=eps, weight_decay=wd)
    g = torch.Generator().manual_seed(1)
    w, m, v = 0.7, 0.0, 0.0
    for e in range(n_epoch):
        for s in range(steps):
            r = rows[e * steps + s].double().tolist()
            t = e * steps + s + 1
            assert opt.state.get(p, {}).get("step", 0) == t - 1
            assert r[6] == pytest.approx(lr / (1 - betas[0] ** t), rel=1e-7)
            assert r[7] == pytest.approx(1 / math.sqrt(1 - betas[1] ** t), rel=1e-7)
            assert r[8] == (1.0 if t == 1 else 0.0)
            assert (r[0], r[1], r[2], r[3], r[4], r[5]) == pytest.approx(
                (1 - lr * wd, betas[0], 1 - betas[0], betas[1], 1 - betas[1], eps), rel=1e-7)
            grad = float(torch.randn(1, generator=g))
            p.grad = torch.tensor([grad], dtype=torch.float64)
            opt.step()
            m0, v0 = (0.0, 0.0) if r[8] else (m, v)       # the first step ignores the stored moments
            m = r[1] * m0 + r[2] * grad
            v = r[3] * v0 + r[4] * grad * grad
            w = w * r[0] - r[6] * m / (math.sqrt(v) * r[7] + r[5])
            assert w == pytest.approx(float(p.detach()), rel=1e-6, abs=1e-9)


def test_portable_trainer_is_torch_adamw():
    torch.manual_seed(0)
    X, y = shard(1, 24)
    eng = FederatedEngine(MLP2(10, 16, 1), "cpu", backend="nccl", loss="mse")
    ref = MLP2(10, 16, 1)
    ref.load_state_dict(eng.model.state_dict())
    torch.manual_seed(7)
    eng.trainer.run(X, y, n_epoch=2, lr=0.01, batch_size=8, weight_decay=0.1, optimizer="adamw", betas=(0.8, 0.9),
                    eps=1e-6)
    torch.manual_seed(7)
    run_local_sgd(ref, X, y, n_epoch=2, lr=0.01, batch_size=8, weight_decay=0.1, loss="mse", optimizer="adamw",
                  betas=(0.8, 0.9), eps=1e-6)
    for (n, a), b in zip(eng.model.named_parameters(), ref.parameters()):
        assert torch.allclose(a, b, atol=1e-6), n


def test_adamw_engine_logical_clients_matches_hand_written():
    """4 logical clients, 2 sampled per round, 3 rounds, full-batch local steps."""
    eng, init = make_engine(4, 2, 3)
    rounds = [eng.run_round(lambda cid: shard(cid, 16 + 8 * cid), n_epoch=EPOCHS).participants for _ in range(3)]
    err = global_error(eng, init, rounds, lambda cid: shard(cid, 16 + 8 * cid))
    assert err < 2e-5, err


def test_adamw_two_gloo_ranks():
    port = 29400 + ((os.getpid() + 431) % 500)
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2",
           "--master-addr", "127.0.0.1", "--master-port", str(port), os.path.join(ROOT, "tests", "mp_adamw_gloo.py")]
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="", OMP_NUM_THREADS="1")
    proc = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=300, cwd=ROOT, env=env)
    tail = "\n".join(proc.stdout.splitlines()[-40:])
    assert proc.returncode == 0 and "RESULT PASS" in proc.stdout, tail
