"""Robust aggregation on the CPU: ``robust_combine`` against numpy / scipy and its exact rules, the configuration and
its rejections, the ``http`` manager plane under a poisoned upload, the seated plan, and a gloo run of the engine."""
import argparse
import asyncio
import os
import subprocess
import sys
from types import SimpleNamespace

import numpy as np
import pytest
import torch
from scipy import stats

from baton_b200.config import FederationConfig
from baton_b200.models import MLP2
from baton_b200.parallel.aggregate import robust_into
from baton_b200.parallel.engine import FederatedEngine
from baton_b200.parallel.robust import RobustConfig, robust_combine

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _bits(t):
    return t.contiguous().view(torch.int32)


@pytest.mark.parametrize("P", [1, 2, 3, 8, 31, 32])
@pytest.mark.parametrize("beta", [0.0, 0.1, 0.25, 0.49])
def test_robust_combine_matches_numpy_and_scipy(P, beta):
    rng = np.random.default_rng(P)
    x = rng.standard_normal((P, 513)).astype(np.float32)
    t = torch.from_numpy(x)
    med = robust_combine(t, RobustConfig("median")).double().numpy()
    np.testing.assert_allclose(med, np.median(x.astype(np.float64), axis=0), rtol=1e-6, atol=1e-6)
    tm = robust_combine(t, RobustConfig("trimmed_mean", beta)).double().numpy()
    np.testing.assert_allclose(tm, stats.trim_mean(x.astype(np.float64), beta, axis=0), rtol=1e-5, atol=1e-6)


def test_exact_rules():
    x = torch.tensor([[4.0], [1.0], [3.0], [2.0]])
    assert float(robust_combine(x, RobustConfig("median"))) == 2.5          # numpy's even median, not torch's 2.0
    assert float(robust_combine(x[:3], RobustConfig("median"))) == 3.0
    # b = floor(beta P): P = 10, beta = 0.1 -> b = 1; beta = 0.19 -> b = 1; beta = 0.2 -> b = 2
    y = torch.arange(10, dtype=torch.float32).unsqueeze(1) ** 2
    for beta, b in ((0.1, 1), (0.19, 1), (0.2, 2), (0.0, 0)):
        cfg = RobustConfig("trimmed_mean", beta)
        assert cfg.trim_count(10) == b
        acc = torch.zeros(1)
        for j in range(b, 10 - b):
            acc = acc + y[j]
        assert torch.equal(robust_combine(y, cfg), acc / (10 - 2 * b))
    # P = 0: no change; P = 1: the client's own delta
    assert torch.equal(robust_combine(torch.zeros(0, 5), RobustConfig("median")), torch.zeros(5))
    one = torch.randn(1, 7)
    for cfg in (RobustConfig("median"), RobustConfig("trimmed_mean", 0.4)):
        assert torch.equal(robust_combine(one, cfg), one[0])


def test_nonfinite_clients_rank_last():
    """P = 5, median, two NaN clients: the result is the 3rd of (finite..., NaN, NaN) in the total order."""
    x = torch.tensor([[1.0, -2.0, float("inf")], [float("nan")] * 3, [0.5, 7.0, 3.0], [float("nan")] * 3,
                      [-1.0, 1.0, float("-inf")]])
    got = robust_combine(x, RobustConfig("median"))
    assert torch.equal(got, torch.tensor([1.0, 7.0, float("inf")]))
    tm = robust_combine(x, RobustConfig("trimmed_mean", 0.2))            # b = 1: drops the lowest and one NaN
    assert torch.isnan(tm).all()
    # -0 < +0 in the order, and every NaN payload is one value
    z = torch.tensor([[-0.0], [0.0], [-0.0]])
    assert _bits(robust_combine(z, RobustConfig("median"))).item() == _bits(torch.tensor([-0.0])).item()


def test_config_validation_and_cli():
    for bad in (("median", -0.1), ("trimmed_mean", 0.5), ("trimmed_mean", float("nan")), ("mode", 0.1)):
        with pytest.raises(ValueError):
            RobustConfig(*bad)
    for bad in ({"aggregator": "max"}, {"aggregator": "trimmed_mean", "trim_ratio": 0.5},
                {"aggregator": "median", "dp_clip": 1.0}):
        with pytest.raises(ValueError):
            FederationConfig(**bad)
    cfg = FederationConfig(aggregator="trimmed_mean", trim_ratio=0.25)
    back = FederationConfig.from_json(cfg.to_json())
    assert back.robust_config() == RobustConfig("trimmed_mean", 0.25)
    assert FederationConfig().robust_config() is None
    parser = argparse.ArgumentParser()
    FederationConfig.add_arguments(parser)
    got = FederationConfig.from_args(parser.parse_args(["--aggregator", "median", "--trim-ratio", "0.3"]))
    assert (got.aggregator, got.trim_ratio) == ("median", 0.3)
    from baton_b200.demo import main as demo_main, make_app
    with pytest.raises(SystemExit):
        demo_main(["manager", "127.0.0.1:1", "1", "--aggregator", "mode"])
    exp = make_app("manager", "127.0.0.1:1", 1, FederationConfig(aggregator="median"))["manager"].experiments[0]
    assert exp.robust == RobustConfig("median") and exp.plane.robust == exp.robust


def test_engine_and_session_reject_excluded_combinations():
    def eng(**kw):
        return FederatedEngine(MLP2(4, 4, 1), "cpu", backend="nccl", loss="mse", **kw)
    for kw in ({"dp_clip": 1.0}, {"scaffold": True}, {"mode": "weights"}, {"tile_flags": True},
               {"trim_ratio": 0.6}, {"logical_clients": 40}, {"logical_clients": 64, "sample_k": 33}):
        with pytest.raises(ValueError):
            eng(aggregator="median", **kw)
    e = eng(aggregator="median", logical_clients=64, sample_k=32)
    assert e.session.max_clients == 32
    e = eng(aggregator="trimmed_mean", logical_clients=16, sample_k=8)
    assert e.session.max_clients == 8
    from baton_b200.parallel.arena import ParamArena
    from baton_b200.parallel.dp import DPConfig
    from baton_b200.parallel.fedavg import NcclSession
    arena = ParamArena(MLP2(4, 4, 1), "cpu")
    for kw in ({"dp": DPConfig(1.0)}, {"scaffold": True}, {"mode": "weights"}, {"tile_flags": True},
               {"max_clients": 33}):
        with pytest.raises(ValueError):
            NcclSession(arena, wire_dtype="fp32", robust=RobustConfig("median"), **kw)
    with pytest.raises(ValueError):
        NcclSession(arena, wire_dtype="fp32", max_clients=2)
    with pytest.raises(ValueError):
        NcclSession(arena, wire_dtype="fp32").aggregate(my_n=1.0, n_clients=1)


def _poisoned_uploads(model, n=5, scale=1e6):
    torch.manual_seed(0)
    ups = []
    for k in range(n):
        c = MLP2(6, 5, 3)
        c.load_state_dict(model.state_dict())
        with torch.no_grad():
            for p in c.parameters():
                p.add_(torch.randn_like(p) * 0.1 * (scale if k == 2 else 1.0))
        ups.append({"state_dict": {n_: t.clone() for n_, t in c.state_dict().items()}, "n_samples": 10 * (k + 1)})
    return ups


@pytest.mark.parametrize("aggregator", ["median", "trimmed_mean", "mean"])
def test_http_plane_round_with_a_poisoned_client(aggregator):
    from baton_b200.parallel.dataplane import make_manager_plane
    torch.manual_seed(1)
    model = MLP2(6, 5, 3)
    before = {n: t.clone() for n, t in model.state_dict().items()}
    ups = _poisoned_uploads(model)
    honest = [u for k, u in enumerate(ups) if k != 2]
    cfg = RobustConfig(aggregator, 0.2) if aggregator != "mean" else None
    plane = make_manager_plane("http", robust=cfg)
    ok = asyncio.run(plane.aggregate(SimpleNamespace(model=model), {str(i): u for i, u in enumerate(ups)}))
    assert ok
    for n, t in model.state_dict().items():
        lo = torch.stack([u["state_dict"][n] for u in honest]).min(0).values
        hi = torch.stack([u["state_dict"][n] for u in honest]).max(0).values
        inside = bool(((t >= lo - 1e-6) & (t <= hi + 1e-6)).all())
        if aggregator == "mean":
            assert not inside, n              # the poisoned average leaves the honest range: the test has teeth
            want = sum(u["state_dict"][n] * u["n_samples"] for u in ups) / sum(u["n_samples"] for u in ups)
            assert torch.allclose(t, want, rtol=1e-5, atol=1e-3)
        else:
            assert inside, n
            stack = torch.stack([u["state_dict"][n].float().flatten() - before[n].flatten() for u in ups])
            assert torch.equal(t.flatten(), before[n].flatten() + robust_combine(stack, cfg))


def test_robust_into_skips_nothing_and_needs_clients():
    model = MLP2(6, 5, 3)
    sd = {n: t.clone() for n, t in model.state_dict().items()}
    assert not robust_into(sd, [], RobustConfig("median"))
    with pytest.raises(ValueError):
        robust_into(sd, [sd] * 33, RobustConfig("median"))


def test_seated_plan_carries_robust():
    from baton_b200.parallel.dataplane import SeatedManagerPlane, SeatedWorkerPlane
    cfg = RobustConfig("trimmed_mean", 0.25)
    cm = SimpleNamespace(clients={"a": {"rank": 0}, "b": {"rank": 1}})
    plane = SeatedManagerPlane("fused", world_size=2, robust=cfg)
    plan = plane.rank_weights(SimpleNamespace(client_manager=cm),
                              {"a": {"n_samples": 128, "rank": 0}, "b": {"n_samples": 64, "rank": 1}})
    assert plan["robust"] == {"kind": "trimmed_mean", "trim_ratio": 0.25}
    assert plan["n_samples_by_rank"] == [128.0, 64.0]
    assert "robust" not in SeatedManagerPlane("fused", world_size=2).rank_weights(
        SimpleNamespace(client_manager=cm), {"a": {"n_samples": 1, "rank": 0}})
    seen = {}

    class Session:
        rank = 0

        def aggregate(self, n, alive, **kw):
            seen.update(kw, n=n)
    SeatedWorkerPlane(Session()).aggregate(None, dict(plan, round=2))
    assert seen["robust"] == cfg and seen["n"] == [128.0, 64.0]


def test_single_process_engine_logical_clients_equals_robust_combine():
    """4 logical clients on one CPU process (nccl session, world 1): the round is robust_combine over the individually
    trained clients' fp32 deltas."""
    from baton_b200.train import run_local_sgd
    torch.manual_seed(0)
    model = MLP2(10, 8, 1)
    eng = FederatedEngine(model, "cpu", backend="nccl", loss="mse", lr=0.05, batch_size=16, wire_dtype="fp32",
                          logical_clients=4, aggregator="median")
    g0 = eng.arena.global_w.clone()

    def shard(cid):
        gen = torch.Generator().manual_seed(100 + cid)
        X = torch.randn(16, 10, generator=gen)
        return X, X.sum(1, keepdim=True) * (cid + 1) * (100.0 if cid == 3 else 1.0)
    deltas = []
    for cid in range(4):
        ref = MLP2(10, 8, 1)
        ref.load_state_dict(model.state_dict())
        X, y = shard(cid)
        run_local_sgd(ref, X, y, n_epoch=1, lr=0.05, batch_size=16, loss="mse")
        deltas.append(torch.cat([p.detach().flatten() for p in ref.parameters()]))
    eng.run_round(shard, n_epoch=1)
    n_p = deltas[0].numel()
    want = g0[:n_p] + robust_combine(torch.stack([d - g0[:n_p] for d in deltas]), RobustConfig("median"))
    assert torch.allclose(eng.arena.global_w[:n_p], want, rtol=0, atol=1e-6)


def test_federated_engine_gloo_ranks_robust_rounds():
    port = 29400 + ((os.getpid() + 611) % 500)
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "3",
           "--master-addr", "127.0.0.1", "--master-port", str(port), os.path.join(ROOT, "tests", "mp_robust_gloo.py")]
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="", OMP_NUM_THREADS="1")
    proc = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=300, cwd=ROOT, env=env)
    tail = "\n".join(proc.stdout.splitlines()[-40:])
    assert proc.returncode == 0 and "RESULT PASS" in proc.stdout, tail
