"""Secure aggregation on one H100: the standalone encode kernel against the numpy reference bit for bit (0..7 peers,
ragged sizes, several keys and nonces, the RFC 8439 keystream), world-1 fused secure rounds against the host reference
(plain, with a server optimizer, with folded logical clients), the register use of the new kernels, and a ResNet-18
engine that learns with ``secure_agg=True``."""
import os
import re
import struct
import subprocess

import numpy as np
import pytest
import torch

from baton_b200.parallel import secagg as sa
from baton_b200.parallel.secagg import SecAggConfig

DEV = "cuda:0"
BF16 = torch.bfloat16
pytestmark = pytest.mark.gpu
RFC_KEY = list(struct.unpack("<8I", bytes(range(32))))


def _keys(n, seed):
    rng = np.random.default_rng(seed)
    return [[int(x) for x in rng.integers(0, 2 ** 32, 8, dtype=np.uint64)] for _ in range(n)]


def _encode_dev(theta, glob, w, R, f, peers, nonce, counter0=0):
    from baton_b200.ops import functional as F
    out = torch.empty(theta.numel(), dtype=torch.int32, device=DEV)
    sat = torch.zeros(1, dtype=torch.int64, device=DEV)
    F.secagg_encode(theta, glob, w, R, f, [k for k, _ in peers], [s for _, s in peers], nonce, counter0, out, sat)
    torch.cuda.synchronize()
    return out.cpu().numpy().view(np.uint32), int(sat.item())


@pytest.mark.parametrize("n_peers", range(8))
@pytest.mark.parametrize("n", [16, 1000, 4099, 65536 + 36])
def test_encode_kernel_matches_reference(n_peers, n):
    rng = np.random.default_rng(n + n_peers)
    th = (rng.standard_normal(n) * 3).astype(np.float32)
    gl = (rng.standard_normal(n)).astype(np.float32)
    th[:: 97] = 1e4                                  # clamped
    if n > 40:
        th[5], th[17], th[33] = np.nan, np.inf, -np.inf
    R = 4.0
    f = sa.frac_bits(R)
    w = float(np.float32(3.0) * (np.float32(1.0) / np.float32(11.0)))
    for trial in range(2):
        keys = _keys(n_peers, 10 * n_peers + trial)
        peers = [(k, 1 if (p + trial) % 2 else -1) for p, k in enumerate(keys)]
        nonce = [1234 + 3 * trial, trial, 7]
        x = (th - gl).astype(np.float32)
        q, sat = sa.encode(x, w, R, f)
        ref = sa.mask(q, peers, nonce, counter0=trial)
        got, gsat = _encode_dev(torch.from_numpy(th).to(DEV), torch.from_numpy(gl).to(DEV), w, R, f, peers, nonce,
                                counter0=trial)
        assert np.array_equal(got, ref), (n_peers, n, trial, int(np.argmax(got != ref)))
        assert gsat == sat


def test_encode_kernel_rfc8439_keystream():
    # x = 0 with one added peer: the upload is the keystream itself
    z = torch.zeros(32, device=DEV)
    got, _ = _encode_dev(z, None, 1.0, 64.0, 24, [(RFC_KEY, 1)], [0x09000000, 0x4A000000, 0], counter0=1)
    assert got[:16].tobytes() == bytes.fromhex("10f1e7e4d13b5915500fdd1fa32071c4c7d1f4c733c068030422aa9ac3d46c4e"
                                               "d2826446079faa0914c2d705d98b02a2b5129cd1de164eb9cbd083e8a2503c4e")
    pt = (b"Ladies and Gentlemen of the class of '99: If I could offer you only one tip for the future, "
          b"sunscreen would be it.")
    got, _ = _encode_dev(torch.zeros(30, device=DEV), None, 1.0, 64.0, 24, [(RFC_KEY, 1)], [0, 0x4A000000, 0],
                         counter0=1)
    ct = bytes(p ^ k for p, k in zip(pt, got.tobytes()))
    assert ct.hex().startswith("6e2e359a2568f98041ba0728dd0d6981e97e7aec1d4360c20a27afccfd9fae0bf91b65c552")
    assert ct.hex().endswith("5af90bbf74a35be6b40b8eedf2785e42874d")


# ---------------------------------------------------------------- world-1 fused rounds
class _Net(torch.nn.Module):
    def __init__(self):
        super().__init__()
        self.fc1 = torch.nn.Linear(72, 250)
        self.bn = torch.nn.BatchNorm1d(250)
        self.fc2 = torch.nn.Linear(250, 6)


def _arena(seed=0):
    from baton_b200.parallel.arena import ParamArena
    torch.manual_seed(seed)
    return ParamArena(_Net(), DEV, momentum=True)


def _session(arena, **kw):
    from baton_b200.parallel.fedavg import FedAvgSession
    return FedAvgSession(arena, wire_dtype="fp32", mode="delta", n_ctas=kw.pop("n_ctas", 8), nvls=False, **kw)


@pytest.mark.parametrize("n_ctas", [1, 8, 132])
def test_fused_round_matches_reference(n_ctas):
    arena = _arena()
    cfg = SecAggConfig(2.0)
    sess = _session(arena, secagg=cfg, n_ctas=n_ctas)
    for rnd in range(3):
        g0 = arena.global_w.clone()
        gen = torch.Generator(device=DEV).manual_seed(rnd)
        delta = torch.randn(arena.n, device=DEV, generator=gen) * (0.5 if rnd else 3.0)
        arena.theta.copy_(g0 + delta)
        src = (arena.theta - g0).cpu().numpy()
        sess.aggregate(my_n=5.0 + rnd)
        torch.cuda.synchronize()
        sess.check()
        d, sat = sa.reference_round([src], [5.0 + rnd], cfg.range, {}, [0, 0, 0])
        ref = (g0.cpu().numpy() + d).astype(np.float32)
        assert np.array_equal(arena.global_w.cpu().numpy().view(np.int32), ref.view(np.int32)), rnd
        assert torch.equal(arena.theta, arena.global_w)
        assert torch.equal(arena.theta_bf16, arena.global_w.to(BF16)) if arena.theta_bf16 is not None else True
        assert not arena.momentum.any()
        assert sess.last_secagg_saturation() == sat
        if rnd == 0:
            assert sat > 0


@pytest.mark.parametrize("kind", ["avgm", "adam"])
def test_fused_round_with_server_optimizer(kind):
    from baton_b200.parallel.server_opt import ServerOptConfig, apply_update_
    arena = _arena(1)
    so = ServerOptConfig(kind, lr=0.05)
    sess = _session(arena, secagg=SecAggConfig(), server_opt=so)
    x = arena.global_w.clone()
    m, v = so.init_state(arena.n_param, DEV)
    for rnd in range(3):
        g0 = arena.global_w.clone()
        delta = torch.randn(arena.n, device=DEV, generator=torch.Generator(device=DEV).manual_seed(20 + rnd)) * 0.02
        arena.theta.copy_(g0 + delta)
        src = (arena.theta - g0).cpu().numpy()
        sess.aggregate(my_n=3.0)
        torch.cuda.synchronize()
        d, _ = sa.reference_round([src], [3.0], 64.0, {}, [0, 0, 0])
        apply_update_(x, torch.from_numpy(d).to(DEV), arena.n_param, m, v, so)
        assert torch.equal(arena.global_w.view(torch.int32), x.view(torch.int32)), (kind, rnd)
        sm, sv = sess.server_state()
        assert torch.equal(sm, m) and (sv is None or torch.equal(sv, v))


def test_fused_round_with_folded_logical_clients():
    from baton_b200.ops import functional as F
    arena = _arena(2)
    sess = _session(arena, secagg=SecAggConfig())
    g0 = arena.global_w.clone()
    acc = torch.zeros_like(arena.theta)
    ns = [64.0, 96.0, 32.0]
    for j, nk in enumerate(ns):
        arena.theta.copy_(g0 + torch.randn(arena.n, device=DEV, generator=torch.Generator(device=DEV).manual_seed(j)))
        F.fold_client(acc, arena.theta, arena.global_w, nk, first=j == 0, reset=j + 1 < len(ns),
                      w_bf16=arena.theta_bf16, momentum=arena.momentum)
    F.fold_finish(acc, arena.theta, arena.global_w, sum(ns))
    src = (arena.theta - g0).cpu().numpy()
    sess.aggregate(my_n=sum(ns))
    torch.cuda.synchronize()
    d, _ = sa.reference_round([src], [sum(ns)], 64.0, {}, [0, 0, 0])
    assert np.array_equal(arena.global_w.cpu().numpy(), (g0.cpu().numpy() + d).astype(np.float32))


def test_fused_round_without_participant_changes_nothing():
    arena = _arena(3)
    sess = _session(arena, secagg=SecAggConfig())
    g0 = arena.global_w.clone()
    arena.theta.copy_(g0 + 1.0)
    sess.aggregate(my_n=0.0)
    torch.cuda.synchronize()
    assert torch.equal(arena.global_w, g0) and torch.equal(arena.theta, g0)


def test_round_arguments_rejected():
    arena = _arena(4)
    sess = _session(arena, secagg=SecAggConfig(), tile_elems=1000)       # not a multiple of 16
    with pytest.raises(RuntimeError):
        sess.aggregate(my_n=1.0)


def test_new_kernels_do_not_spill():
    """Compile fedavg.cu with -Xptxas -v: the secure instantiations stay under the collective's 96-register cap
    without spilling, and the standalone encode kernel does not spill."""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    from baton_b200.build_ext import NVCC_FLAGS, _nvcc
    out = "/tmp/secagg_spill_{}.o".format(os.getpid())
    proc = subprocess.run([_nvcc(), *NVCC_FLAGS, "-c", os.path.join(root, "baton_b200", "csrc", "fedavg.cu"), "-o", out],
                          stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if os.path.exists(out):
        os.remove(out)
    assert proc.returncode == 0, proc.stdout[-2000:]
    found = 0
    for m in re.finditer(r"Compiling entry function '(\w+)'.*?\n(.*?)Used (\d+) registers", proc.stdout, re.S):
        if "SecAgg" in m.group(1) or "secagg" in m.group(1):
            found += 1
            assert "0 bytes spill stores" in m.group(2), m.group(1)
            assert int(m.group(3)) <= 96, m.group(1)
    assert found == 3, found


# ---------------------------------------------------------------- ResNet-18 engine
def _colour_shard(n, seed, noise=1.0):
    colours = torch.randn(10, 3, generator=torch.Generator().manual_seed(100)) * 0.5
    g = torch.Generator().manual_seed(seed)
    y = torch.randint(0, 10, (n,), generator=g)
    X = colours[y][:, None, None, :] + noise * torch.randn(n, 32, 32, 3, generator=g)
    return X.to(DEV).to(BF16), y.to(DEV)


# Held-out accuracy threshold as in the mixing and clipping tests (chance is 0.1); a plain fp32-wire engine reaches
# well above it on this task.
SECAGG_MIN_ACC = 0.6


def test_resnet18_engine_learns_with_secure_aggregation():
    from baton_b200.models import resnet18
    from baton_b200.parallel.engine import FederatedEngine
    torch.manual_seed(0)
    eng = FederatedEngine(resnet18(10), DEV, backend="fused", lr=0.05, batch_size=128, n_ctas=64, seed=4,
                          wire_dtype="fp32", secure_agg=True)
    assert not eng.prepack and not eng.session.use_nvls
    X, y = _colour_shard(2048, seed=1)
    Xh, yh = _colour_shard(1024, seed=2)
    for _ in range(4):
        eng.run_round((X, y), n_epoch=1)
        assert eng.last_secagg_saturation() == 0
    res = eng.evaluate((Xh, yh))
    print("held-out accuracy after 4 secure rounds: {:.4f}".format(res.accuracy))
    assert res.accuracy >= SECAGG_MIN_ACC, res


def test_resnet18_engine_secure_rounds_with_logical_clients_and_server_opt():
    from baton_b200.models import resnet18
    from baton_b200.parallel.engine import FederatedEngine
    torch.manual_seed(0)
    eng = FederatedEngine(resnet18(10), DEV, backend="fused", lr=0.05, batch_size=128, n_ctas=64, seed=3,
                          wire_dtype="fp32", secure_agg=True, logical_clients=3, sample_k=2, server_opt="avgm",
                          server_lr=1.0)
    data = {c: _colour_shard(384 + 64 * c, seed=c) for c in range(3)}
    hist = []
    for _ in range(3):
        hist += eng.run_round(lambda cid: data[cid], n_epoch=1).loss_history
    eng.sync()
    torch.cuda.synchronize()
    assert hist and all(np.isfinite(hist)), hist
    assert torch.isfinite(eng.arena.global_w).all()


@pytest.mark.multigpu
def test_multi_gpu_against_nccl_and_reference():
    import sys
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    n = min(torch.cuda.device_count(), 8)
    port = 29500 + ((os.getpid() + 977) % 1000)
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(n),
           "--master-addr", "127.0.0.1", "--master-port", str(port), os.path.join(root, "tests", "mp_secagg_check.py")]
    proc = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=900, cwd=root)
    tail = "\n".join(proc.stdout.splitlines()[-60:])
    assert proc.returncode == 0 and "RESULT PASS" in proc.stdout, tail
