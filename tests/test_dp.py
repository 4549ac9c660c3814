"""DP-FedAvg, CPU tier: the host Philox sampler, the RDP accountant, the manager-side estimator, an engine round on two
gloo ranks against the estimator computed by hand, and the configuration."""
import argparse
import math
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from baton_b200.config import FederationConfig
from baton_b200.models import LinearModel, MLP2
from baton_b200.parallel.aggregate import dp_fedavg_into
from baton_b200.parallel.dp import (DPConfig, RDPAccountant, normals, philox4x32_10, rdp_sampled_gaussian)
from baton_b200.parallel.engine import FederatedEngine
from conftest import run_async
from fedtest import Federation

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("ctr,key,want", [
    ([0, 0, 0, 0], (0, 0), [0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8]),
    ([0xffffffff] * 4, (0xffffffff, 0xffffffff), [0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd]),
    ([0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344], (0xa4093822, 0x299f31d0),
     [0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1]),
])
def test_host_philox_reproduces_the_random123_known_answers(ctr, key, want):
    got = philox4x32_10(np.array(ctr, dtype=np.uint32), key)
    assert [int(x) for x in got] == want


def test_host_normals_are_standard_normal_and_index_addressed():
    from scipy import stats
    z = normals(0x1234_5678_9abc_def0, 7, 10 ** 6)
    assert abs(z.mean()) < 5e-3 and abs(z.std() - 1.0) < 5e-3
    assert stats.kstest(z, "norm").pvalue > 1e-3
    # a pure function of the element index: any window equals the same slice of the whole stream
    assert np.array_equal(normals(0x1234_5678_9abc_def0, 7, 13, start=5), z[5:18])
    assert not np.array_equal(normals(0x1234_5678_9abc_def0, 8, 16), z[:16])


def test_rdp_full_participation_is_the_gaussian_closed_form():
    for sigma in (0.5, 1.0, 3.0):
        for alpha in (1.5, 2.0, 7.0, 32.0):
            assert rdp_sampled_gaussian(1.0, sigma, alpha) == pytest.approx(alpha / (2 * sigma ** 2), rel=1e-12)
    acc = RDPAccountant(2.0, orders=(4.0,))
    acc.step(1.0, rounds=10)
    assert acc.rdp()[0] == pytest.approx(10 * 4.0 / 8.0)


def _rdp_by_quadrature(q, sigma, alpha):
    from scipy import integrate
    # A_alpha = E_{x ~ N(0, s^2)} [((1 - q) + q exp((2x - 1) / (2 s^2)))^alpha]
    def f(x):      # in log space: the likelihood ratio overflows far in the tail, where the density has long vanished
        log_lr = np.logaddexp(math.log1p(-q), math.log(q) + (2 * x - 1) / (2 * sigma ** 2))
        return math.exp(-x * x / (2 * sigma ** 2) + alpha * log_lr) / (math.sqrt(2 * math.pi) * sigma)
    a, _ = integrate.quad(f, -np.inf, np.inf, epsabs=0, epsrel=1e-12, limit=500)
    return math.log(a) / (alpha - 1)


@pytest.mark.parametrize("q", [0.01, 0.1, 0.5])
@pytest.mark.parametrize("sigma", [0.7, 1.0, 4.0])
def test_rdp_sampled_gaussian_matches_the_defining_integral(q, sigma):
    for alpha in (1.5, 2.0, 3.0, 4.5, 8.0):
        want = _rdp_by_quadrature(q, sigma, alpha)
        assert rdp_sampled_gaussian(q, sigma, alpha) == pytest.approx(want, rel=1e-6), (q, sigma, alpha)


def test_epsilon_grows_with_rounds_and_shrinks_with_noise():
    def eps(sigma, rounds, q=0.25):
        a = RDPAccountant(sigma)
        a.step(q, rounds)
        return a.get_privacy_spent(1e-5)[0]
    assert eps(1.0, 10) < eps(1.0, 100) < eps(1.0, 1000)
    assert eps(4.0, 100) < eps(1.0, 100) < eps(0.7, 100)
    zero = RDPAccountant(0.0)
    zero.step(1.0)
    assert math.isinf(zero.get_privacy_spent(1e-5)[0])


def test_dp_fedavg_into_matches_the_estimator_in_float64():
    torch.manual_seed(0)
    g = MLP2(6, 5, 3)
    clients = []
    for k in range(4):
        c = MLP2(6, 5, 3)
        c.load_state_dict(g.state_dict())
        with torch.no_grad():
            for p in c.parameters():
                p.add_(torch.randn_like(p) * (0.3 * (k + 1)))
        clients.append({n: t.clone() for n, t in c.state_dict().items()})
    with torch.no_grad():
        clients[2]["fc1.weight"][0, 0] = float("nan")        # a poisoned update: s = 0, still counts in m
    gsd = {n: t.clone() for n, t in g.state_dict().items()}
    before = {n: t.clone().double() for n, t in gsd.items()}
    C, sigma, seed, rnd = 1.5, 0.8, 99, 3
    factors = dp_fedavg_into(gsd, clients, clip=C, noise_multiplier=sigma, seed=seed, round_index=rnd)
    keys = list(before)
    deltas = [torch.cat([(c[k].double() - before[k]).flatten() for k in keys]) for c in clients]
    want_s = []
    for d in deltas:
        nrm = float(d.norm())
        want_s.append(0.0 if not math.isfinite(nrm) else min(1.0, C / nrm))
    assert factors == pytest.approx(want_s, rel=1e-12) and factors[2] == 0.0 and 0.0 < min(factors[:2]) < 1.0
    total = sum(s * d for s, d in zip(want_s, deltas) if s != 0.0)
    z = torch.from_numpy(normals(seed, rnd, total.numel()))
    want = torch.cat([before[k].flatten() for k in keys]) + (total + sigma * C * z) / 4
    got = torch.cat([gsd[k].double().flatten() for k in keys])
    assert torch.allclose(got, want, rtol=0, atol=1e-6)


def test_federated_engine_two_gloo_ranks_dp_round():
    port = 29400 + ((os.getpid() + 353) % 500)
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2",
           "--master-addr", "127.0.0.1", "--master-port", str(port), os.path.join(ROOT, "tests", "mp_dp_gloo.py")]
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="", OMP_NUM_THREADS="1")
    proc = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=300, cwd=ROOT, env=env)
    tail = "\n".join(proc.stdout.splitlines()[-40:])
    assert proc.returncode == 0 and "RESULT PASS" in proc.stdout, tail


def test_engine_single_process_logical_clients_dp_and_accountant():
    """One CPU process, 4 logical clients: the round equals the uniform mean of the individually clipped deltas plus
    the noise, and the accountant composes one round at q = 1."""
    torch.manual_seed(0)
    model = MLP2(10, 8, 1)
    eng = FederatedEngine(model, "cpu", backend="nccl", loss="mse", lr=0.05, batch_size=16, wire_dtype="fp32",
                          logical_clients=4, dp_clip=0.05, dp_noise_multiplier=0.5, dp_seed=5)
    g0 = eng.arena.global_w.clone()

    def shard(cid):
        gen = torch.Generator().manual_seed(100 + cid)
        X = torch.randn(16, 10, generator=gen)
        return X, X.sum(1, keepdim=True) * (cid + 1)
    # the clients' trained replicas, computed the same way the engine trains them
    deltas = []
    for cid in range(4):
        ref = MLP2(10, 8, 1)
        ref.load_state_dict(model.state_dict())
        from baton_b200.train import run_local_sgd
        X, y = shard(cid)
        run_local_sgd(ref, X, y, n_epoch=1, lr=0.05, batch_size=16, loss="mse")
        deltas.append(torch.cat([p.detach().flatten() for p in ref.parameters()]))
    eng.run_round(shard, n_epoch=1)
    n_p = deltas[0].numel()
    w0 = g0[:n_p].double()
    ds = [d.double() - w0 for d in deltas]
    s = [min(1.0, 0.05 / float(d.norm())) for d in ds]
    assert eng.last_clip_factors() == pytest.approx(s, rel=1e-5)
    z = torch.from_numpy(normals(5, 0, eng.arena.n))[:n_p]
    want = w0 + (sum(si * d for si, d in zip(s, ds)) + 0.5 * 0.05 * z) / 4
    assert torch.allclose(eng.arena.global_w[:n_p].double(), want, rtol=0, atol=2e-6)
    eps, order = eng.privacy_spent(1e-5)
    assert math.isfinite(eps) and eps > 0
    assert eng.accountant.history == {1.0: 1}


def test_dp_arguments_are_validated():
    with pytest.raises(ValueError):
        FederatedEngine(MLP2(4, 4, 1), "cpu", backend="nccl", loss="mse", dp_clip=-1.0)
    with pytest.raises(ValueError):
        FederatedEngine(MLP2(4, 4, 1), "cpu", backend="nccl", loss="mse", dp_noise_multiplier=1.0)   # C = 0
    with pytest.raises(ValueError):
        FederatedEngine(MLP2(4, 4, 1), "cpu", backend="nccl", loss="mse", mode="weights", dp_clip=1.0)
    with pytest.raises(ValueError):
        DPConfig(float("nan"), 1.0)
    eng = FederatedEngine(MLP2(4, 4, 1), "cpu", backend="nccl", loss="mse")
    assert eng.dp is None and eng.last_clip_factors() == []
    with pytest.raises(RuntimeError):
        eng.privacy_spent(1e-5)


def test_http_manager_plane_aggregates_with_dp_fedavg():
    """The manager's tensor plane with ``dp``: the global model becomes the DP-FedAvg of the uploads (uniform over the
    participants, whatever their sample counts), the factors are kept, and the noise stream advances per round."""
    import asyncio
    from types import SimpleNamespace
    from baton_b200.parallel.dataplane import HttpManagerPlane
    torch.manual_seed(0)
    model = MLP2(6, 5, 3)
    uploads = []
    for k in range(3):
        c = MLP2(6, 5, 3)
        c.load_state_dict(model.state_dict())
        with torch.no_grad():
            for p in c.parameters():
                p.add_(torch.randn_like(p) * 0.5)
        uploads.append({"state_dict": {n: t.clone() for n, t in c.state_dict().items()}, "n_samples": 10 * (k + 1)})
    dp = DPConfig(1.0, 0.5, seed=21)
    plane = HttpManagerPlane(dp=dp)
    for rnd in range(2):
        want = {n: t.clone() for n, t in model.state_dict().items()}
        factors = dp_fedavg_into(want, [u["state_dict"] for u in uploads], clip=1.0, noise_multiplier=0.5, seed=21,
                                 round_index=rnd)
        ok = asyncio.run(plane.aggregate(SimpleNamespace(model=model), {str(i): u for i, u in enumerate(uploads)}))
        assert ok and plane.last_clip_factors == factors and max(factors) < 1.0
        for n, t in model.state_dict().items():
            assert torch.equal(t, want[n]), n


def test_http_manager_plane_skips_clients_that_trained_nothing():
    import asyncio
    from types import SimpleNamespace
    from baton_b200.parallel.dataplane import HttpManagerPlane
    model = MLP2(6, 5, 3)
    sd = {n: t.clone() for n, t in model.state_dict().items()}
    plane = HttpManagerPlane(dp=DPConfig(1.0, 0.5, seed=2))
    ok = asyncio.run(plane.aggregate(SimpleNamespace(model=model), {"a": {"state_dict": sd, "n_samples": 0}}))
    assert not ok and plane.dp_rounds == 0 and plane.last_clip_factors == []


def test_config_json_and_cli_round_trip_dp():
    cfg = FederationConfig(dp_clip=1.0, dp_noise_multiplier=0.5, dp_seed=7, dp_delta=1e-6)
    back = FederationConfig.from_json(cfg.to_json())
    assert (back.dp_clip, back.dp_noise_multiplier, back.dp_seed, back.dp_delta) == (1.0, 0.5, 7, 1e-6)
    assert back.dp_config() == DPConfig(1.0, 0.5, seed=7)
    d = FederationConfig()
    assert (d.dp_clip, d.dp_noise_multiplier, d.dp_delta, d.dp_seed) == (0.0, 0.0, 1e-5, None)
    assert d.dp_config() is None
    parser = argparse.ArgumentParser()
    FederationConfig.add_arguments(parser)
    got = FederationConfig.from_args(parser.parse_args(["--dp-clip", "2", "--dp-noise-multiplier", "1.5",
                                                        "--dp-seed", "3", "--dp-delta", "1e-6"]))
    assert (got.dp_clip, got.dp_noise_multiplier, got.dp_seed, got.dp_delta) == (2.0, 1.5, 3, 1e-6)
    for bad in ({"dp_clip": -1.0}, {"dp_clip": float("inf")}, {"dp_noise_multiplier": 1.0},
                {"dp_clip": 1.0, "dp_noise_multiplier": float("nan")}, {"dp_delta": 0.0}, {"dp_delta": 1.0}):
        with pytest.raises(ValueError):
            FederationConfig(**bad)
    from baton_b200.demo import main as demo_main
    for argv in (["--dp-noise-multiplier", "1.0"], ["--dp-clip=-0.5"], ["--dp-clip", "1", "--dp-delta", "2"]):
        with pytest.raises(SystemExit):
            demo_main(["manager", "127.0.0.1:1", "1"] + argv)


def test_demo_manager_builder_carries_dp():
    from baton_b200.demo import make_app
    app = make_app("manager", "127.0.0.1:1", 1, FederationConfig(dp_clip=0.5, dp_noise_multiplier=1.0, dp_seed=4,
                                                                 dp_delta=1e-6))
    exp = app["manager"].experiments[0]
    assert exp.dp == DPConfig(0.5, 1.0, seed=4) and exp.dp_delta == 1e-6 and exp.plane.dp == exp.dp


def test_seated_plan_counts_clients_and_carries_dp():
    from types import SimpleNamespace
    from baton_b200.parallel.dataplane import SeatedManagerPlane, SeatedWorkerPlane
    dp = DPConfig(0.3, 2.0, seed=0xABCDEF)
    cm = SimpleNamespace(clients={"a": {"rank": 0}, "b": {"rank": 1}, "c": {"rank": 2}})
    plane = SeatedManagerPlane("fused", world_size=3, dp=dp)
    plan = plane.rank_weights(SimpleNamespace(client_manager=cm),
                              {"a": {"n_samples": 128, "rank": 0}, "b": {"n_samples": 512, "rank": 1},
                               "c": {"n_samples": 0, "rank": 2}})
    assert plan["n_samples_by_rank"] == [1.0, 1.0, 0.0]             # clients, not samples
    assert plan["dp"] == {"clip": 0.3, "noise_multiplier": 2.0, "seed": 0xABCDEF}
    plain = SeatedManagerPlane("fused", world_size=3).rank_weights(
        SimpleNamespace(client_manager=cm), {"a": {"n_samples": 128, "rank": 0}})
    assert plain["n_samples_by_rank"] == [128.0, 0.0, 0.0] and "dp" not in plain
    seen = {}

    class Session:
        rank = 1

        def aggregate(self, n, alive, **kw):
            seen.update(kw, n=n, alive=alive)
    SeatedWorkerPlane(Session()).aggregate(None, dict(plan, round=5))
    assert seen["dp"] == dp and seen["round_index"] == 5 and seen["n"] == [1.0, 1.0, 0.0]


@run_async
async def test_http_round_with_a_dp_manager_reports_epsilon():
    from baton_b200.demo import LinearTestWorker
    fed = Federation()
    dp = DPConfig(0.05, 1.0, seed=9)
    exp = await fed.start_manager(LinearModel(), dp=dp, dp_delta=1e-5)
    try:
        before = {n: t.detach().clone() for n, t in exp.model.state_dict().items()}
        for seed in (11, 12):
            await fed.add_worker(cls=LinearTestWorker, seed=seed, train_kwargs={"lr": 0.02})
        status, _ = await fed.get("start_round?n_epoch=4")
        assert status == 200
        await fed.wait_round_closed()
        assert exp.update_manager.n_updates == 1
        assert len(exp.plane.last_clip_factors) == 2 and max(exp.plane.last_clip_factors) < 1.0
        delta = torch.cat([(t.detach() - before[n]).flatten() for n, t in exp.model.state_dict().items()])
        assert float(delta.norm()) > 0.0
        status, metrics = await fed.get("metrics")
        assert status == 200
        m = metrics["dp"]
        assert m["rounds"] == 1 and m["clip"] == 0.05 and m["noise_multiplier"] == 1.0 and m["delta"] == 1e-5
        assert math.isfinite(m["epsilon"]) and m["epsilon"] > 0 and m["clipped_fraction"] == 1.0
    finally:
        await fed.close()
