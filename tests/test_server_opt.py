"""Server-side optimizers (parallel/server_opt.py) on the CPU: the host step against numpy formulas, the FedAvg identity,
zero-weight rounds, validation, NcclSession / the engine on a CPU arena, FederationConfig and the demo flags, the
``http`` manager plane through a Manager with CPU workers against a host replay, checkpoint save / resume, the seated
planes' rejection, and a 2-process gloo run (``tests/mp_server_opt_gloo.py``)."""
import math

import numpy as np
import pytest
import torch

from baton_b200.parallel.arena import ParamArena
from baton_b200.parallel.fedavg import NcclSession
from baton_b200.parallel.robust import RobustConfig
from baton_b200.parallel.server_opt import KINDS, ServerOptConfig, apply_update_, server_step_


def _np_step(kind, x, d, m, v, c):
    """The table of parallel/server_opt.py in numpy fp32, one rounded operation at a time."""
    b1, omb1, b2, omb2, lr, tau = (np.float32(t) for t in c)
    if kind == "avgm":
        m = np.add(np.multiply(b1, m), d)
        return np.add(x, np.multiply(lr, m)), m, v
    m = np.add(np.multiply(b1, m), np.multiply(omb1, d))
    dd = np.multiply(d, d)
    if kind == "adagrad":
        v = np.add(v, dd)
    elif kind == "yogi":
        v = np.subtract(v, np.multiply(np.multiply(omb2, dd), np.sign(np.subtract(v, dd))))
    else:
        v = np.add(np.multiply(b2, v), np.multiply(omb2, dd))
    return np.add(x, np.divide(np.multiply(lr, m), np.add(np.sqrt(v), tau))), m, v


@pytest.mark.parametrize("kind", KINDS)
def test_step_matches_numpy_over_five_rounds(kind):
    cfg = ServerOptConfig(kind, lr=0.3, b1=0.8, b2=0.95, tau=0.05)
    g = torch.Generator().manual_seed(1)
    n = 257
    x = torch.randn(n, generator=g)
    m, v = cfg.init_state(n, "cpu")
    xn, mn = x.numpy().copy(), m.numpy().copy()
    vn = v.numpy().copy() if v is not None else None
    with np.errstate(all="ignore"):
        for r in range(5):
            d = torch.randn(n, generator=g) * (0.5 ** r)
            d[:7] = 0.0                                   # zeros
            d[7:20] = -d[7:20].abs()                      # negatives
            if r == 3 and v is not None:                  # Yogi: v - d*d changes sign for some elements
                d[20:40] = v[20:40].sqrt() * 1.5
            xn, mn, vn = _np_step(kind, xn, d.numpy(), mn, vn, cfg.coefficients())
            server_step_(x, d, m, v, cfg)
            assert np.array_equal(x.numpy(), xn) and np.array_equal(m.numpy(), mn)
            if v is not None:
                assert np.array_equal(v.numpy(), vn)
    if kind == "yogi":
        assert (v > 0).all()


def test_yogi_sign_flips_both_ways():
    cfg = ServerOptConfig("yogi", lr=1.0, b2=0.5, tau=1.0)       # v starts at 1
    x = torch.zeros(3)
    m, v = cfg.init_state(3, "cpu")
    server_step_(x, torch.tensor([2.0, 0.5, 1.0]), m, v, cfg)   # d*d = 4 > v, 0.25 < v, 1 == v
    assert v.tolist() == [1.0 + 0.5 * 4.0, 1.0 - 0.5 * 0.25, 1.0]


def test_coefficients_are_fp32_of_fp64():
    cfg = ServerOptConfig("adam", lr=0.01, b1=0.9, b2=0.99, tau=1e-3)
    want = [float(np.float32(t)) for t in (0.9, 1.0 - 0.9, 0.99, 1.0 - 0.99, 0.01, 1e-3)]
    assert list(cfg.coefficients()) == want
    assert cfg.v0() == float(np.float32(1e-3 * 1e-3))
    assert ServerOptConfig("avgm", lr=1.0).init_state(8, "cpu")[1] is None


def test_avgm_identity_is_plain_add():
    cfg = ServerOptConfig("avgm", lr=1.0, b1=0.0)
    g = torch.Generator().manual_seed(2)
    x = torch.randn(1000, generator=g)
    ref = x.clone()
    m, v = cfg.init_state(1000, "cpu")
    for _ in range(3):
        d = torch.randn(1000, generator=g)
        server_step_(x, d, m, v, cfg)
        ref.add_(d)
        assert torch.equal(x, ref)


def test_apply_update_buffers_take_plain_add():
    cfg = ServerOptConfig("adam", lr=0.1)
    x = torch.randn(24)
    d = torch.randn(24)
    m, v = cfg.init_state(16, "cpu")
    x0 = x.clone()
    apply_update_(x, d, 16, m, v, cfg)
    assert torch.equal(x[16:], x0[16:] + d[16:])
    assert not torch.equal(x[:16], x0[:16] + d[:16])


@pytest.mark.parametrize("bad", [
    dict(kind="sgd", lr=1.0), dict(kind="adam", lr=None), dict(kind="adam", lr=0.0), dict(kind="adam", lr=-1.0),
    dict(kind="adam", lr=math.inf), dict(kind="adam", lr=math.nan), dict(kind="adam", lr=1.0, tau=0.0),
    dict(kind="adam", lr=1.0, tau=math.inf), dict(kind="adam", lr=1.0, b1=1.0), dict(kind="adam", lr=1.0, b1=-0.1),
    dict(kind="adam", lr=1.0, b2=1.0), dict(kind="adam", lr=1.0, b2=math.nan)])
def test_validation(bad):
    with pytest.raises(ValueError):
        ServerOptConfig(**bad)


def test_dict_round_trip():
    cfg = ServerOptConfig("yogi", lr=0.02, b1=0.5, b2=0.9, tau=1e-2)
    assert ServerOptConfig.from_dict(cfg.to_dict()) == cfg


class _Net(torch.nn.Module):
    def __init__(self):
        super().__init__()
        self.fc = torch.nn.Linear(6, 5)
        self.bn = torch.nn.BatchNorm1d(5)

    def forward(self, x):
        return self.bn(self.fc(x))


def _arena():
    torch.manual_seed(0)
    return ParamArena(_Net(), torch.device("cpu"), momentum=True)


def _perturb(a, seed):
    g = torch.Generator().manual_seed(seed)
    a.theta.add_(torch.randn(a.n, generator=g) * 0.1)


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("robust", [None, RobustConfig("median")])
def test_nccl_session_steps_with_the_oracle(kind, robust):
    cfg = ServerOptConfig(kind, lr=0.5)
    a = _arena()
    s = NcclSession(a, wire_dtype="fp32", server_opt=cfg, robust=robust)
    x = a.global_w.clone()
    m, v = cfg.init_state(a.n_param, "cpu")
    for r in range(3):
        _perturb(a, 10 + r)
        d = (a.theta - a.global_w).clone()
        s.aggregate(my_n=4.0)
        apply_update_(x, d, a.n_param, m, v, cfg)
        assert torch.equal(a.global_w, x) and torch.equal(a.theta, x)
        sm, sv = s.server_state()
        assert torch.equal(sm, m) and (v is None or torch.equal(sv, v))
    assert a.nbytes()["server_m"] == a.n_param * 4
    assert ("server_v" in a.nbytes()) == cfg.needs_v


def test_zero_weight_round_is_a_noop():
    cfg = ServerOptConfig("adam", lr=0.5)
    a = _arena()
    s = NcclSession(a, wire_dtype="fp32", server_opt=cfg)
    _perturb(a, 3)
    s.aggregate(my_n=1.0)
    g0, (m0, v0) = a.global_w.clone(), [t.clone() for t in s.server_state()]
    _perturb(a, 4)
    s.aggregate(my_n=0.0)
    m1, v1 = s.server_state()
    assert torch.equal(a.global_w, g0) and torch.equal(m1, m0) and torch.equal(v1, v0)


def test_avgm_identity_session_equals_plain_session():
    a, b = _arena(), _arena()
    sa = NcclSession(a, wire_dtype="bf16", server_opt=ServerOptConfig("avgm", lr=1.0, b1=0.0))
    sb = NcclSession(b, wire_dtype="bf16")
    for r in range(3):
        _perturb(a, 20 + r)
        _perturb(b, 20 + r)
        sa.aggregate(my_n=2.0)
        sb.aggregate(my_n=2.0)
        assert torch.equal(a.global_w, b.global_w)


def test_sessions_reject_weights_mode_and_bad_types():
    with pytest.raises(ValueError, match="delta"):
        NcclSession(_arena(), mode="weights", server_opt=ServerOptConfig("adam", lr=1.0))
    with pytest.raises(TypeError):
        NcclSession(_arena(), server_opt="adam")
    with pytest.raises(RuntimeError):
        NcclSession(_arena()).server_state()


def test_engine_options():
    from baton_b200.parallel.engine import FederatedEngine
    with pytest.raises(ValueError, match="server_lr"):
        FederatedEngine(_Net(), "cpu", backend="nccl", server_opt="adam")
    with pytest.raises(ValueError, match="delta"):
        FederatedEngine(_Net(), "cpu", backend="nccl", server_opt="adam", server_lr=1.0, mode="weights")
    with pytest.raises(ValueError):
        FederatedEngine(_Net(), "cpu", backend="nccl", server_opt="lamb", server_lr=1.0)
    eng = FederatedEngine(_Net(), "cpu", backend="nccl", server_opt="yogi", server_lr=0.1, server_betas=(0.5, 0.9),
                          server_tau=1e-2)
    assert eng.session.server_opt == ServerOptConfig("yogi", 0.1, 0.5, 0.9, 1e-2)
    m, v = eng.server_state()
    assert m.numel() == eng.arena.n_param and torch.all(v == ServerOptConfig("yogi", 0.1, tau=1e-2).v0())
    with pytest.raises(RuntimeError):
        FederatedEngine(_Net(), "cpu", backend="nccl").server_state()


# ---------------------------------------------------------------- configuration, CLI, manager planes, checkpoints
def test_federation_config_and_demo_flags():
    import argparse

    from baton_b200.config import FederationConfig
    assert FederationConfig().server_opt_config() is None
    cfg = FederationConfig(server_opt="adam", server_lr=0.02, server_beta1=0.8, server_beta2=0.95, server_tau=1e-2)
    assert cfg.server_opt_config() == ServerOptConfig("adam", 0.02, 0.8, 0.95, 1e-2)
    assert FederationConfig.from_json(cfg.to_json()) == cfg
    for bad in (dict(server_opt="adam"), dict(server_opt="lamb", server_lr=1.0),
                dict(server_opt="yogi", server_lr=1.0, server_beta2=1.0),
                dict(server_opt="avgm", server_lr=-1.0), dict(server_opt="adam", server_lr=1.0, server_tau=0.0)):
        with pytest.raises(ValueError):
            FederationConfig(**bad)
    with pytest.raises(ValueError, match="http plane"):
        FederationConfig(server_opt="adam", server_lr=1.0, backend="fused")
    p = argparse.ArgumentParser()
    FederationConfig.add_arguments(p)
    ns = p.parse_args(["--server-opt", "yogi", "--server-lr", "0.05", "--server-beta1", "0.5",
                       "--server-beta2", "0.9", "--server-tau", "0.01"])
    assert FederationConfig.from_args(ns).server_opt_config() == ServerOptConfig("yogi", 0.05, 0.5, 0.9, 0.01)


def test_seated_planes_reject_server_opt():
    from baton_b200.parallel.dataplane import SeatedManagerPlane, make_manager_plane
    cfg = ServerOptConfig("adam", lr=0.1)
    for spec in ("fused", "nccl", SeatedManagerPlane("fused")):
        with pytest.raises(ValueError, match="stale m and v"):
            make_manager_plane(spec, server_opt=cfg)
    from aiohttp import web

    from baton_b200.control import Manager
    from baton_b200.models import LinearModel
    with pytest.raises(ValueError, match="stale m and v"):
        Manager(web.Application()).register_experiment(LinearModel(), dataplane="nccl", server_opt=cfg)


def _uploads(model, rnd, n=3, rel=0.01):
    """Client state_dicts within 1 % of the global model (same sign, within a factor 2): the mean, and d = scratch -
    live, are then exact in the sense of Sterbenz's lemma."""
    g = torch.Generator().manual_seed(500 + rnd)
    ups = {}
    for k in range(n):
        sd = {name: (t * (1.0 + rel * torch.rand(t.shape, generator=g)) if t.is_floating_point() else t + k)
              for name, t in model.state_dict().items()}
        ups[str(k)] = {"state_dict": sd, "n_samples": 8 * (k + 1)}
    return ups


def _net():
    torch.manual_seed(3)
    net = _Net()
    with torch.no_grad():                       # buffers away from zero so the relative uploads move them
        net.bn.running_mean.fill_(0.5)
    return net


def test_http_plane_avgm_identity_equals_fedavg_into():
    import asyncio
    from types import SimpleNamespace

    from baton_b200.parallel.aggregate import fedavg_into
    from baton_b200.parallel.dataplane import make_manager_plane
    a, b = _net(), _net()
    plane = make_manager_plane("http", server_opt=ServerOptConfig("avgm", lr=1.0, b1=0.0))
    for rnd in range(3):
        ups = _uploads(a, rnd)
        assert asyncio.run(plane.aggregate(SimpleNamespace(model=a), ups))
        ref = b.state_dict()
        assert fedavg_into(ref, [u["state_dict"] for u in ups.values()], [u["n_samples"] for u in ups.values()])
        for k, t in a.state_dict().items():
            assert torch.equal(t, ref[k]), k


def _replay(model, rounds, cfg):
    """Host replay of the http plane: fedavg_into into a scratch copy, d = scratch - live over the parameters,
    server_step_ there, the aggregate on the buffers."""
    from baton_b200.parallel.aggregate import fedavg_into
    m = v = None
    names = [n for n, _ in model.named_parameters()]
    for ups in rounds:
        live = model.state_dict()
        scratch = {k: t.clone() for k, t in live.items()}
        datas = [u for u in ups.values() if "state_dict" in u]
        if not fedavg_into(scratch, [u["state_dict"] for u in datas], [u["n_samples"] for u in datas]):
            continue
        x = torch.cat([live[n].reshape(-1).float() for n in names])
        d = torch.cat([scratch[n].reshape(-1).float() for n in names]) - x
        if m is None:
            m, v = cfg.init_state(x.numel(), "cpu")
        server_step_(x, d, m, v, cfg)
        off = 0
        with torch.no_grad():
            for n in names:
                scratch[n] = x[off: off + live[n].numel()].view(live[n].shape)
                off += live[n].numel()
            for k, t in live.items():
                t.copy_(scratch[k])
    return m, v


@pytest.mark.parametrize("kind", ["avgm", "adam"])
def test_http_plane_through_manager_equals_host_replay(kind):
    """A Manager with two CPU workers over HTTP for 3 rounds: the global model equals the host replay of the uploads
    the plane received, and /metrics reports the optimizer."""
    import asyncio

    from fedtest import Federation

    from baton_b200.models import LinearModel
    cfg = ServerOptConfig(kind, lr=0.5 if kind == "avgm" else 0.05)

    async def run():
        fed = Federation()
        torch.manual_seed(0)
        exp = await fed.start_manager(LinearModel(), server_opt=cfg)
        start = {k: t.clone() for k, t in exp.model.state_dict().items()}
        seen = []
        orig = exp.plane.aggregate

        async def recording(experiment, responses):
            seen.append({c: dict(d) for c, d in responses.items()})
            return await orig(experiment, responses)
        exp.plane.aggregate = recording
        try:
            await fed.add_worker(n=6, seed=1)
            await fed.add_worker(n=9, seed=2)
            for _ in range(3):
                await fed.get("start_round?n_epoch=2")
                await fed.wait_round_closed()
            status, metrics = await fed.get("metrics")
            assert status == 200 and metrics["server_opt"] == cfg.to_dict()
            return start, seen, {k: t.clone() for k, t in exp.model.state_dict().items()}, exp.plane
        finally:
            await fed.close()

    start, seen, final, plane = asyncio.run(run())
    assert len(seen) == 3
    replay = LinearModel()
    replay.load_state_dict(start)
    m, v = _replay(replay, seen, cfg)
    for k, t in replay.state_dict().items():
        assert torch.equal(final[k], t), k
    assert torch.equal(plane.server_m, m) and (v is None or torch.equal(plane.server_v, v))


def test_http_plane_checkpoint_resume_continues_the_run(tmp_path):
    """Save after 2 rounds, restore into a fresh model and plane, run round 3: equal to 3 uninterrupted rounds.  A
    file without the entry restores the initial state."""
    import asyncio
    from types import SimpleNamespace

    from baton_b200 import ckpt
    from baton_b200.control import UpdateManager
    from baton_b200.parallel.dataplane import make_manager_plane
    cfg = ServerOptConfig("yogi", lr=0.05)
    base = _net()
    rounds = [_uploads(base, r) for r in range(3)]
    full, full_plane = _net(), make_manager_plane("http", server_opt=cfg)
    for ups in rounds:
        assert asyncio.run(full_plane.aggregate(SimpleNamespace(model=full), ups))
    first, plane1 = _net(), make_manager_plane("http", server_opt=cfg)
    for ups in rounds[:2]:
        asyncio.run(plane1.aggregate(SimpleNamespace(model=first), ups))
    path = ckpt.save_checkpoint(str(tmp_path), "exp", first, UpdateManager("exp"), server_opt=plane1.server_state())
    resumed, plane2 = _net(), make_manager_plane("http", server_opt=cfg)
    payload = ckpt.load_checkpoint(path, resumed)
    plane2.load_server_state(payload["server_opt"])
    assert asyncio.run(plane2.aggregate(SimpleNamespace(model=resumed), rounds[2]))
    for k, t in resumed.state_dict().items():
        assert torch.equal(t, full.state_dict()[k]), k
    assert torch.equal(plane2.server_m, full_plane.server_m) and torch.equal(plane2.server_v, full_plane.server_v)
    stock = torch.load(path, weights_only=True)["state_dict"]      # the stock layout is unchanged
    _Net().load_state_dict(stock)
    plain = ckpt.save_checkpoint(str(tmp_path / "plain"), "exp", first, UpdateManager("exp"))
    plane2.load_server_state(ckpt.load_checkpoint(plain).get("server_opt"))
    assert plane2.server_m is None and plane2.server_v is None
    with pytest.raises(ValueError, match="differs"):
        make_manager_plane("http", server_opt=ServerOptConfig("adam", lr=0.05)).load_server_state(payload["server_opt"])


def test_manager_resume_restores_the_server_state(tmp_path):
    import asyncio

    from fedtest import Federation

    from baton_b200.models import LinearModel
    cfg = ServerOptConfig("adam", lr=0.05)

    async def run():
        fed = Federation()
        exp = await fed.start_manager(LinearModel(), checkpoint_dir=str(tmp_path), server_opt=cfg)
        try:
            await fed.add_worker(n=5, seed=3)
            await fed.get("start_round?n_epoch=1")
            await fed.wait_round_closed()
            for _ in range(500):
                if exp.last_checkpoint:
                    break
                await asyncio.sleep(0.01)
            assert exp.last_checkpoint
            saved = (exp.plane.server_m.clone(), exp.plane.server_v.clone(),
                     {k: t.clone() for k, t in exp.model.state_dict().items()})
        finally:
            await fed.close()
        fed2 = Federation()
        exp2 = await fed2.start_manager(LinearModel(), checkpoint_dir=str(tmp_path), resume=True, server_opt=cfg)
        try:
            assert torch.equal(exp2.plane.server_m, saved[0]) and torch.equal(exp2.plane.server_v, saved[1])
            for k, t in exp2.model.state_dict().items():
                assert torch.equal(t, saved[2][k])
        finally:
            await fed2.close()
    asyncio.run(run())


def test_nccl_sessions_on_gloo_stay_bitwise_equal():
    import os
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    port = 29400 + ((os.getpid() + 811) % 500)
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2",
           "--master-addr", "127.0.0.1", "--master-port", str(port),
           os.path.join(root, "tests", "mp_server_opt_gloo.py")]
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="", OMP_NUM_THREADS="1")
    proc = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=300, cwd=root,
                          env=env)
    tail = "\n".join(proc.stdout.splitlines()[-40:])
    assert proc.returncode == 0 and "RESULT PASS" in proc.stdout, tail
