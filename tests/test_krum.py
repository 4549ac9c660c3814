"""Multi-Krum on the CPU: ``krum_select`` against a brute-force scipy reference and its exact rules, the configuration
and its rejections, the ``http`` manager plane under a model-poisoning attack, the seated plan, the engine on one
process and a gloo run of the engine (``tests/mp_krum_gloo.py``)."""
import argparse
import asyncio
import os
import subprocess
import sys
from types import SimpleNamespace

import numpy as np
import pytest
import torch
from scipy.spatial.distance import cdist

from baton_b200.config import FederationConfig
from baton_b200.models import MLP2
from baton_b200.parallel.engine import FederatedEngine
from baton_b200.parallel.robust import RobustConfig, krum_select, robust_combine

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INF = float("inf")


def _reference(x: np.ndarray, f: int, m):
    """Brute force: scipy's squared distances, k smallest per row, lexicographic (score, position) order."""
    p = x.shape[0]
    D = cdist(x.astype(np.float64), x.astype(np.float64), "sqeuclidean")
    D[~np.isfinite(D)] = INF
    k = min(max(1, p - f - 2), p - 1)
    scores = [float(sum(sorted(D[i, j] for j in range(p) if j != i)[:k])) for i in range(p)]
    keep = min(max(m if m is not None else p - f, 1), p)
    order = sorted(range(p), key=lambda i: (scores[i], i))[:keep]
    return D, np.array(scores), np.isin(np.arange(p), order)


@pytest.mark.parametrize("P,f,m", [(3, 0, None), (5, 1, None), (7, 2, None), (7, 2, 1), (12, 3, 4), (32, 4, None)])
def test_krum_select_matches_scipy(P, f, m):
    rng = np.random.default_rng(P + 10 * f)
    x = (rng.standard_normal((P, 301)) * rng.uniform(0.5, 3.0, (P, 1))).astype(np.float32)
    cfg = RobustConfig("krum", krum_f=f, krum_m=m)
    D, scores, kept = krum_select(torch.from_numpy(x), cfg)
    rD, rs, rk = _reference(x, f, m)
    np.testing.assert_allclose(D.numpy(), rD, rtol=1e-12, atol=1e-9)
    np.testing.assert_allclose(scores.numpy(), rs, rtol=1e-12)
    assert kept.tolist() == rk.tolist()
    got = robust_combine(torch.from_numpy(x), cfg)
    assert torch.equal(got, robust_combine(torch.from_numpy(x)[kept], RobustConfig("trimmed_mean", 0.0)))


def test_clamping_tables():
    cfg = RobustConfig("krum", krum_f=2)
    k, m = cfg.krum_tables()
    assert len(k) == len(m) == 33
    # k = max(1, P - f - 2) capped at P - 1; m = clamp(P - f, 1, P)
    assert k[:8] == [0, 0, 1, 1, 1, 1, 2, 3] and m[:8] == [0, 1, 1, 1, 2, 3, 4, 5]
    assert k[32] == 28 and m[32] == 30
    one = RobustConfig("krum", krum_f=1, krum_m=1)
    assert one.krum_tables()[1][1:6] == [1, 1, 1, 1, 1]
    big = RobustConfig("krum", krum_f=0, krum_m=50)            # krum_m > P clamps to P
    assert [big.krum_kept(p) for p in (1, 5, 32)] == [1, 5, 32]
    assert cfg.trim_table() == [0] * 33                         # the kept mean drops nothing


def test_small_rounds_and_ties():
    cfg = RobustConfig("krum", krum_f=1)
    assert torch.equal(robust_combine(torch.zeros(0, 4), cfg), torch.zeros(4))     # P = 0: no change
    one = torch.randn(1, 6)
    D, s, kept = krum_select(one, cfg)
    assert s.tolist() == [0.0] and kept.tolist() == [True]
    assert torch.equal(robust_combine(one, cfg), one[0])
    two = torch.tensor([[1.0, 2.0], [3.0, 5.0]])
    D, s, kept = krum_select(two, cfg)                       # P = 2: k = 1, m = 1, equal scores: first position
    assert D[0, 1] == 13.0 and s.tolist() == [13.0, 13.0] and kept.tolist() == [True, False]
    # exact ties between whole clients are broken by position
    tie = torch.tensor([[0.0], [1.0], [0.0], [1.0], [0.5]])
    D, s, kept = krum_select(tie, RobustConfig("krum", krum_f=0, krum_m=2))
    # k = 3: a 0 / 1 row has 0 (its twin) + 0.25 (the 0.5 row) + 1; the 0.5 row has 3 * 0.25
    assert s.tolist() == [1.25, 1.25, 1.25, 1.25, 0.75]
    assert kept.tolist() == [True, False, False, False, True]


def test_nonfinite_clients_score_inf_and_are_dropped():
    rng = np.random.default_rng(3)
    x = torch.from_numpy(rng.standard_normal((6, 40)).astype(np.float32))
    x[1, 5] = float("nan")
    x[4, 0] = INF
    cfg = RobustConfig("krum", krum_f=2)
    D, s, kept = krum_select(x, cfg)
    assert torch.isinf(D[1]).sum() == 5 and torch.isinf(D[4]).sum() == 5 and D[1, 1] == 0
    assert s[1] == INF and s[4] == INF and torch.isfinite(s[[0, 2, 3, 5]]).all()
    assert kept.tolist() == [True, False, True, True, False, True]
    assert torch.isfinite(robust_combine(x, cfg)).all()


def test_config_validation_and_cli():
    for bad in ({"krum_f": -1}, {"krum_f": 1.5}, {"krum_m": 0}, {"krum_m": 2.0}):
        with pytest.raises(ValueError):
            RobustConfig("krum", **bad)
    for bad in ({"aggregator": "krum", "krum_f": 1, "clients": 4},               # 4 < 2f + 3
                {"aggregator": "krum", "krum_f": 2, "logical_clients": 16, "sample_k": 6},
                {"aggregator": "krum", "krum_m": 0, "clients": 4},
                {"aggregator": "krum", "dp_clip": 1.0, "clients": 4}):
        with pytest.raises(ValueError):
            FederationConfig(**bad)
    cfg = FederationConfig(aggregator="krum", krum_f=2, krum_m=3, logical_clients=16, sample_k=8)
    back = FederationConfig.from_json(cfg.to_json())
    assert back.robust_config() == RobustConfig("krum", 0.1, 2, 3)
    parser = argparse.ArgumentParser()
    FederationConfig.add_arguments(parser)
    got = FederationConfig.from_args(parser.parse_args(
        ["--aggregator", "krum", "--krum-f", "1", "--krum-m", "2", "--clients", "5"]))
    assert (got.aggregator, got.krum_f, got.krum_m) == ("krum", 1, 2)
    assert FederationConfig.from_args(parser.parse_args(["--aggregator", "krum", "--clients", "3"])).krum_m is None
    from baton_b200.demo import main as demo_main, make_app
    with pytest.raises(SystemExit):
        demo_main(["manager", "127.0.0.1:1", "1", "--aggregator", "krum", "--krum-f", "1"])    # 2 clients < 5
    exp = make_app("manager", "127.0.0.1:1", 1, FederationConfig(aggregator="krum", krum_f=1, clients=5))[
        "manager"].experiments[0]
    assert exp.robust == RobustConfig("krum", krum_f=1) and exp.plane.robust == exp.robust


def test_engine_and_session_reject_excluded_combinations():
    def eng(**kw):
        return FederatedEngine(MLP2(4, 4, 1), "cpu", backend="nccl", loss="mse", **kw)
    for kw in ({"dp_clip": 1.0}, {"scaffold": True}, {"mode": "weights"}, {"tile_flags": True},
               {"logical_clients": 40}, {"sample_k": 6, "krum_f": 2}, {"logical_clients": 4, "krum_f": 1},
               {"krum_m": 0}, {"krum_f": -1}):
        with pytest.raises(ValueError):
            eng(aggregator="krum", **dict({"logical_clients": 16}, **kw))
    with pytest.raises(ValueError):
        eng(aggregator="krum")                                       # one client per round < 2f + 3
    e = eng(aggregator="krum", logical_clients=16, sample_k=7, krum_f=2)
    assert e.session.max_clients == 7 and e.robust.kind == "krum"
    from baton_b200.parallel.arena import ParamArena
    from baton_b200.parallel.dp import DPConfig
    from baton_b200.parallel.fedavg import NcclSession
    arena = ParamArena(MLP2(4, 4, 1), "cpu")
    for kw in ({"dp": DPConfig(1.0)}, {"scaffold": True}, {"mode": "weights"}, {"tile_flags": True},
               {"max_clients": 33}):
        with pytest.raises(ValueError):
            NcclSession(arena, wire_dtype="fp32", robust=RobustConfig("krum"), **kw)
    with pytest.raises(RuntimeError):
        NcclSession(arena, wire_dtype="fp32", robust=RobustConfig("krum")).last_krum()


def _uploads(model, n=7, bad=(1, 4), s=10.0):
    """n clients around the global model; the clients in ``bad`` upload -s times a genuine update."""
    torch.manual_seed(0)
    ups = []
    for k in range(n):
        c = MLP2(6, 5, 3)
        c.load_state_dict(model.state_dict())
        with torch.no_grad():
            for p in c.parameters():
                d = 0.05 * torch.randn_like(p) + 0.1                # honest updates share a direction
                p.add_(-s * d if k in bad else d)
        ups.append({"state_dict": {n_: t.clone() for n_, t in c.state_dict().items()}, "n_samples": 10 * (k + 1)})
    return ups


def test_http_plane_rejects_scaled_sign_flipped_uploads():
    from baton_b200.parallel.dataplane import make_manager_plane
    torch.manual_seed(1)
    model = MLP2(6, 5, 3)
    before = {n: t.clone() for n, t in model.state_dict().items()}
    ups = _uploads(model)
    cfg = RobustConfig("krum", krum_f=2)
    keys = list(before)
    flat = torch.stack([torch.cat([u["state_dict"][k].float().flatten() - before[k].flatten() for k in keys])
                        for u in ups])
    kept = krum_select(flat, cfg)[2]
    assert kept.tolist() == [True, False, True, True, False, True, True]      # both attackers rejected
    plane = make_manager_plane("http", robust=cfg)
    ok = asyncio.run(plane.aggregate(SimpleNamespace(model=model), {str(i): u for i, u in enumerate(ups)}))
    assert ok
    honest = [u for k, u in enumerate(ups) if kept[k]]
    for n, t in model.state_dict().items():
        stack = torch.stack([u["state_dict"][n].float().flatten() - before[n].flatten() for u in honest])
        assert torch.equal(t.flatten(), before[n].flatten() + robust_combine(stack, RobustConfig("trimmed_mean", 0.0)))


def test_seated_plan_carries_krum():
    from baton_b200.parallel.dataplane import SeatedManagerPlane, SeatedWorkerPlane
    cfg = RobustConfig("krum", krum_f=1, krum_m=2)
    assert RobustConfig.from_dict(cfg.to_dict()) == cfg
    assert RobustConfig.from_dict(RobustConfig("krum").to_dict()).krum_m is None
    cm = SimpleNamespace(clients={"a": {"rank": 0}, "b": {"rank": 1}})
    plane = SeatedManagerPlane("fused", world_size=2, robust=cfg)
    plan = plane.rank_weights(SimpleNamespace(client_manager=cm),
                              {"a": {"n_samples": 128, "rank": 0}, "b": {"n_samples": 64, "rank": 1}})
    assert plan["robust"] == {"kind": "krum", "f": 1, "m": 2}
    seen = {}

    class Session:
        rank = 0

        def aggregate(self, n, alive, **kw):
            seen.update(kw, n=n)
    SeatedWorkerPlane(Session()).aggregate(None, dict(plan, round=2))
    assert seen["robust"] == cfg and seen["n"] == [128.0, 64.0]


def test_single_process_engine_and_last_krum():
    """7 logical clients on one CPU process: the round is krum over the individually trained clients' fp32 deltas,
    and last_krum maps the scores to client ids."""
    from baton_b200.train import run_local_sgd
    torch.manual_seed(0)
    model = MLP2(10, 8, 1)
    eng = FederatedEngine(model, "cpu", backend="nccl", loss="mse", lr=0.05, batch_size=16, wire_dtype="fp32",
                          logical_clients=7, aggregator="krum", krum_f=2)
    g0 = eng.arena.global_w.clone()

    def shard(cid):
        gen = torch.Generator().manual_seed(100 + cid)
        X = torch.randn(16, 10, generator=gen)
        return X, X.sum(1, keepdim=True) * (-50.0 if cid in (2, 5) else 1.0)
    deltas = []
    for cid in range(7):
        ref = MLP2(10, 8, 1)
        ref.load_state_dict(model.state_dict())
        X, y = shard(cid)
        run_local_sgd(ref, X, y, n_epoch=1, lr=0.05, batch_size=16, loss="mse")
        deltas.append(torch.cat([p.detach().flatten() for p in ref.parameters()]))
    eng.run_round(shard, n_epoch=1)
    n_p = deltas[0].numel()
    stack = torch.stack([d - g0[:n_p] for d in deltas])
    D, scores, kept = krum_select(stack, RobustConfig("krum", krum_f=2))
    assert kept.tolist() == [True, True, False, True, True, False, True]
    want = g0[:n_p] + robust_combine(stack, RobustConfig("krum", krum_f=2))
    assert torch.allclose(eng.arena.global_w[:n_p], want, rtol=0, atol=1e-6)
    rep = eng.last_krum()
    assert sorted(rep) == list(range(7))
    assert [rep[c][1] for c in range(7)] == kept.tolist()
    np.testing.assert_allclose([rep[c][0] for c in range(7)], scores.numpy(), rtol=1e-4)


def test_federated_engine_gloo_ranks_krum_rounds():
    port = 29400 + ((os.getpid() + 733) % 500)
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "3",
           "--master-addr", "127.0.0.1", "--master-port", str(port), os.path.join(ROOT, "tests", "mp_krum_gloo.py")]
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="", OMP_NUM_THREADS="1")
    proc = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=300, cwd=ROOT, env=env)
    tail = "\n".join(proc.stdout.splitlines()[-40:])
    assert proc.returncode == 0 and "RESULT PASS" in proc.stdout, tail
