"""Server-side optimizers on the GPU: the *_sopt instantiations of the fused collective against the host step
(parallel/server_opt.py) bit for bit where the aggregate is reproducible on the host, FedAvgM(1, 0) against the plain
instantiations for every kind of round and wire, DP / SCAFFOLD / fp8 against NcclSession, invariance to the CTA count
and the tiling, the arrival flags, and ResNet-18 engine rounds."""
import os
import subprocess
import sys

import pytest
import torch

from baton_b200.parallel.robust import RobustConfig, krum_select, robust_combine
from baton_b200.parallel.server_opt import KINDS, ServerOptConfig, apply_update_

BF16 = torch.bfloat16
DEV = "cuda:0"
pytestmark = pytest.mark.gpu
MEAN = RobustConfig("trimmed_mean", 0.0)


def _bits(t):
    return t.contiguous().view(torch.int32)


class _Net(torch.nn.Module):
    """Parameters followed by float buffers (BatchNorm running statistics) and an integer one."""
    def __init__(self):
        super().__init__()
        self.fc1 = torch.nn.Linear(72, 250)
        self.bn = torch.nn.BatchNorm1d(250)
        self.fc2 = torch.nn.Linear(250, 6)


def _arena(seed=0):
    from baton_b200.parallel.arena import ParamArena
    torch.manual_seed(seed)
    a = ParamArena(_Net(), DEV, momentum=True)
    assert a.n > a.n_param
    return a


def _session(arena, wire, **kw):
    from baton_b200.parallel.fedavg import FedAvgSession
    return FedAvgSession(arena, wire_dtype=wire, mode="delta", n_ctas=kw.pop("n_ctas", 8), nvls=False, **kw)


def _deltas(n, S, seed):
    gen = torch.Generator(device=DEV).manual_seed(seed)
    common = torch.randn(n, device=DEV, generator=gen) * 0.01
    return [common + torch.randn(n, device=DEV, generator=gen) * 0.004 * (1 + 0.45 * j) for j in range(S)]


def _decoded(x, wire):
    return x.to(BF16).float() if wire == "bf16" else x.clone()


def _round(arena, sess, deltas, robust):
    """One round from the replicas g0 + delta_j; returns the host-reproducible aggregate d."""
    g0 = arena.global_w.clone()
    ups = [_decoded(g0 + dl - g0, sess.wire_dtype) for dl in deltas]      # what the pack uploads
    if robust is None:
        arena.theta.copy_(g0 + deltas[0])
        sess.aggregate(my_n=1.0)
        d = ups[0]
    else:
        for j, dl in enumerate(deltas):
            arena.theta.copy_(g0 + dl)
            sess.pack_client(j, reset=j + 1 < len(deltas))
        sess.aggregate(my_n=float(len(deltas)), n_clients=len(deltas))
        stack = torch.stack(ups)
        if robust.kind == "krum":
            stack, robust = stack[krum_select(stack, robust)[2].to(DEV)], MEAN
        d = _decoded(robust_combine(stack, robust), sess.wire_dtype)
    torch.cuda.synchronize()
    sess.check()
    return g0, d


AGGS = {"plain": None, "median": RobustConfig("median"), "krum": RobustConfig("krum", krum_f=1)}


@pytest.mark.parametrize("wire", ["fp32", "bf16"])
@pytest.mark.parametrize("agg", list(AGGS))
@pytest.mark.parametrize("kind", KINDS)
def test_world1_kernel_equals_the_host_step(kind, agg, wire):
    cfg = ServerOptConfig(kind, lr=0.3 if kind == "avgm" else 0.01, b1=0.9, b2=0.99, tau=1e-3)
    robust = AGGS[agg]
    S = 1 if robust is None else 5
    arena = _arena(1)
    kw = {} if robust is None else {"robust": robust, "max_clients": S}
    sess = _session(arena, wire, server_opt=cfg, **kw)
    x = arena.global_w.cpu()
    m, v = cfg.init_state(arena.n_param, "cpu")
    npar = arena.n_param
    for r in range(3):
        g0, d = _round(arena, sess, _deltas(arena.n, S, seed=10 * r + S), robust)
        apply_update_(x, d.cpu(), npar, m, v, cfg)
        got_m, got_v = sess.server_state()
        assert torch.equal(_bits(got_m.cpu()), _bits(m)), r
        if v is not None:
            assert torch.equal(_bits(got_v.cpu()), _bits(v)), r
        else:
            assert got_v is None
        assert torch.equal(_bits(arena.global_w.cpu()), _bits(x)), r
        assert torch.equal(_bits(arena.global_w[npar:]), _bits(g0[npar:] + d[npar:]))     # buffers: global += d
        assert torch.equal(arena.theta, arena.global_w)
        assert torch.equal(arena.theta_bf16, arena.theta.to(BF16))
        assert float(arena.momentum.abs().max()) == 0.0


def _pair_rounds(kind_of_round, wire, rounds=2):
    """The same rounds through a plain session and through one with FedAvgM(lr=1, b1=0)."""
    out = []
    for sopt in (None, ServerOptConfig("avgm", lr=1.0, b1=0.0)):
        arena = _arena(2)
        kw = {"server_opt": sopt}
        robust = None
        if kind_of_round == "dp":
            from baton_b200.parallel.dp import DPConfig
            kw["dp"] = DPConfig(0.05, 0.7, seed=1234)
        elif kind_of_round == "scaffold":
            kw["scaffold"] = True
        elif kind_of_round in ("median", "krum"):
            robust = AGGS[kind_of_round]
            kw.update(robust=robust, max_clients=5)
        sess = _session(arena, wire, **kw)
        c = torch.zeros(arena.n_param, device=DEV)
        for r in range(rounds):
            deltas = _deltas(arena.n, 5 if robust is not None else 1, seed=40 + r)
            if kind_of_round == "scaffold":
                arena.theta.copy_(arena.global_w + deltas[0])
                sess.aggregate(my_n=1.0, control=(c, deltas[0][: arena.n_param] * 3.0, 4))
                torch.cuda.synchronize()
                sess.check()
            else:
                _round(arena, sess, deltas, robust)
        out.append((arena.global_w.clone(), c.clone()))
    return out


@pytest.mark.parametrize("wire", ["fp32", "bf16", "fp8"])
@pytest.mark.parametrize("kind_of_round", ["plain", "dp", "scaffold", "median", "krum"])
def test_avgm_identity_equals_the_plain_instantiation(kind_of_round, wire):
    (g_plain, c_plain), (g_sopt, c_sopt) = _pair_rounds(kind_of_round, wire)
    assert torch.equal(_bits(g_sopt), _bits(g_plain))
    assert torch.equal(_bits(c_sopt), _bits(c_plain))


def _rel(a, b):
    return float((a.double() - b.double()).norm() / b.double().norm().clamp_min(1e-30))


@pytest.mark.parametrize("case", ["dp", "scaffold", "fp8"])
def test_dp_scaffold_fp8_against_nccl_session(case):
    """FedAdam on top of DP (fixed seed), SCAFFOLD and the fp8 wire: the fused collective against NcclSession (fp32
    wire on the host side).  DP's noise is added before the wire cast on the device and after it on the host, and
    fp8 rounds each block to 3 mantissa bits, so the steps agree to a tolerance, not bitwise."""
    from baton_b200.parallel.dp import DPConfig
    from baton_b200.parallel.fedavg import NcclSession
    cfg = ServerOptConfig("adam", lr=0.01)
    steps = []
    for fused in (True, False):
        arena = _arena(3)
        g_init = arena.global_w.clone()
        kw = {"server_opt": cfg}
        if case == "dp":
            kw["dp"] = DPConfig(0.5, 0.3, seed=99)
        if case == "scaffold":
            kw["scaffold"] = True
        wire = "fp8" if case == "fp8" else "fp32"
        sess = _session(arena, wire, **kw) if fused else NcclSession(arena, wire_dtype="fp32", mode="delta", **kw)
        c = torch.zeros(arena.n_param, device=DEV)
        for r in range(3):
            dl = _deltas(arena.n, 1, seed=70 + r)[0]
            arena.theta.copy_(arena.global_w + dl)
            if case == "scaffold":
                sess.aggregate(my_n=1.0, control=(c, dl[: arena.n_param] * 2.0, 2))
            else:
                sess.aggregate(my_n=1.0)
            torch.cuda.synchronize()
            sess.check()
        steps.append((arena.global_w - g_init, c.clone()))
    tol = {"dp": 1e-4, "scaffold": 1e-5, "fp8": 0.08}[case]
    assert _rel(steps[0][0], steps[1][0]) < tol, _rel(steps[0][0], steps[1][0])
    if case == "scaffold":
        assert _rel(steps[0][1], steps[1][1]) < 1e-6


@pytest.mark.parametrize("wire", ["bf16", "fp8"])
def test_result_is_invariant_to_ctas_and_tiles(wire):
    cfg = ServerOptConfig("yogi", lr=0.01)
    res = []
    for n_ctas, tile in ((8, 1024), (132, 4096), (32, 0)):
        arena = _arena(4)
        sess = _session(arena, wire, server_opt=cfg, n_ctas=n_ctas, tile_elems=tile)
        for r in range(2):
            _round(arena, sess, _deltas(arena.n, 1, seed=90 + r), None)
        res.append((arena.global_w.clone(), *[t.clone() for t in sess.server_state()]))
    for other in res[1:]:
        for a, b in zip(other, res[0]):
            assert torch.equal(_bits(a), _bits(b))


def test_arrival_flags_with_fedadam():
    cfg = ServerOptConfig("adam", lr=0.01)
    arena = _arena(5)
    sess = _session(arena, "bf16", server_opt=cfg, tile_flags=True)
    x = arena.global_w.cpu()
    m, v = cfg.init_state(arena.n_param, "cpu")
    for r in range(2):
        _, d = _round(arena, sess, _deltas(arena.n, 1, seed=5 + r), None)
        apply_update_(x, d.cpu(), arena.n_param, m, v, cfg)
        assert torch.equal(_bits(arena.global_w.cpu()), _bits(x))
        assert int(sess.tile_flags.min()) == r + 1 and int(sess.tile_flags.max()) == r + 1


def test_resnet18_engine_fedadam_fused_matches_nccl():
    """Three FedAdam rounds of a ResNet-18 engine on backend='fused' against backend='nccl' (the difference calibrated by
    two fused runs).  After round 1 the BatchNorm running statistics are compared with a plain engine's to a
    TOLERANCE, not bitwise: training accumulates the BatchNorm batch statistics with fp32 atomics, so two plain runs
    already differ in the last bits; the bound is three times that plain/plain spread.  That buffers take exactly
    global += d is checked bitwise at the kernel level (test_world1_kernel_equals_the_host_step)."""
    from baton_b200.models import resnet18
    from baton_b200.parallel.engine import FederatedEngine
    from test_gpu_fedprox import _image_data
    X, y = _image_data(DEV, 512)

    def run(backend, server_opt, rounds):
        torch.manual_seed(0)
        kw = {"server_opt": server_opt, "server_lr": 0.01} if server_opt else {}
        eng = FederatedEngine(resnet18(10), DEV, backend=backend, lr=0.05, batch_size=128, n_ctas=64, **kw)
        g0 = eng.arena.global_w.clone()
        for _ in range(rounds):
            eng.run_round((X, y), n_epoch=1)
        eng.sync()
        torch.cuda.synchronize()
        eng.session.check()
        return eng.arena.global_w - g0, eng.arena.n_param

    a, npar = run("fused", "adam", 3)
    b, _ = run("fused", "adam", 3)
    c, _ = run("nccl", "adam", 3)
    noise, diff = _rel(b, a), _rel(c, a)
    print("3 FedAdam rounds, rel diff: fused/fused {:.2e}, fused/nccl {:.2e}".format(noise, diff))
    assert diff <= 3.0 * noise + 1e-3, (diff, noise)
    p1, _ = run("fused", None, 1)
    p2, _ = run("fused", None, 1)
    s1, _ = run("fused", "adam", 1)
    bn_noise, bn_diff = _rel(p2[npar:], p1[npar:]), _rel(s1[npar:], p1[npar:])
    print("round-1 BatchNorm statistics rel diff: plain/plain {:.2e}, plain/adam {:.2e}".format(bn_noise, bn_diff))
    assert bn_diff <= 3.0 * bn_noise + 1e-6, (bn_diff, bn_noise)


COMBOS = {
    "fedprox": dict(prox_mu=0.05),                      # the proximal anchor is global_w after the server step
    "adamw": dict(optimizer="adamw", lr=1e-3),
    "momentum": dict(momentum=0.9),
    "logical_sample_k": dict(logical_clients=4, sample_k=2),
}


@pytest.mark.parametrize("combo", list(COMBOS))
def test_engine_combinations_fused_match_nccl(combo):
    """FedAdam with FedProx, local AdamW, local momentum, and logical clients sampled 2 of 4: three engine rounds on
    backend='fused' (the one-client rounds take the optimizer-emitted upload) against backend='nccl', fp32 wire."""
    from baton_b200.models import MLP2
    from baton_b200.parallel.engine import FederatedEngine
    gen = torch.Generator().manual_seed(1)
    shards = {}
    for cid in range(4):
        X = torch.randn(128 + 64 * cid, 16, generator=gen)
        shards[cid] = (X.to(DEV), (X @ (torch.arange(1.0, 17.0) * (1 + 0.5 * cid))).unsqueeze(1).to(DEV))
    kw = dict(loss="mse", lr=0.002, batch_size=64, wire_dtype="fp32", seed=11, server_opt="adam", server_lr=0.01)
    kw.update(COMBOS[combo])
    out = {}
    for backend in ("fused", "nccl"):
        torch.manual_seed(0)
        eng = FederatedEngine(MLP2(16, 64, 1), DEV, backend=backend, **kw)
        g0 = eng.arena.global_w.clone()
        for _ in range(3):
            eng.run_round((lambda cid: shards[cid]) if eng.logical_clients else shards[0], n_epoch=2)
        eng.sync()
        torch.cuda.synchronize()
        eng.session.check()
        m, v = eng.server_state()
        out[backend] = (eng.arena.global_w - g0, m.clone(), v.clone())
    (gf, mf, vf), (gn, mn, vn) = out["fused"], out["nccl"]
    assert float(gf.abs().max()) > 0.0
    assert _rel(gf, gn) < 1e-4 and _rel(mf, mn) < 1e-4 and _rel(vf, vn) < 1e-4, (_rel(gf, gn), _rel(mf, mn))


@pytest.mark.multigpu
def test_multi_gpu_against_nccl():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    n = min(torch.cuda.device_count(), 8)
    port = 29500 + ((os.getpid() + 811) % 1000)
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(n),
           "--master-addr", "127.0.0.1", "--master-port", str(port), os.path.join(root, "tests", "mp_server_opt_check.py")]
    proc = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=900, cwd=root)
    tail = "\n".join(proc.stdout.splitlines()[-60:])
    assert proc.returncode == 0 and "RESULT PASS" in proc.stdout, tail
