"""DP-FedAvg on the GPU: the clip-factor kernel, the DP instantiations of the fused collective (clip factors, noise,
invariance to the tiling, the optimizer-emitted upload) and engine rounds with logical clients and with bcast_gemm."""
import math

import pytest
import torch

from baton_b200.parallel.dp import DPConfig, normals

BF16 = torch.bfloat16
DEV = "cuda:0"


def _load():
    from baton_b200.ops import load
    return load()


@pytest.mark.gpu
@pytest.mark.parametrize("n", [1024, 65536 + 8, 3_000_008])
def test_clip_factor_kernel_matches_float64_and_is_deterministic(n):
    from baton_b200.ops import functional as F
    C = _load()
    gen = torch.Generator(device=DEV).manual_seed(n)
    g = torch.randn(n, device=DEV, generator=gen)
    t = g + torch.randn(n, device=DEV, generator=gen) * 1e-3
    work = torch.zeros(C.DP_WORK_WORDS, dtype=torch.int64, device=DEV)
    bad = torch.zeros(1, dtype=torch.int32, device=DEV)
    want_norm = float((t.double() - g.double()).norm())
    outs = []
    for clip in (want_norm / 3, want_norm * 2):
        s, nrm = torch.zeros(1, device=DEV), torch.zeros(1, device=DEV)
        copy = torch.zeros(1, device=DEV)
        F.dp_clip_factor(t, g, clip, work, s, nrm, s_copy_ptr=copy.data_ptr(), nonfinite=bad)
        assert float(nrm) == pytest.approx(want_norm, rel=1e-5)
        assert float(s) == pytest.approx(min(1.0, clip / want_norm), rel=1e-5)
        assert torch.equal(s, copy)
        outs.append((s.clone(), nrm.clone()))
    s2, nrm2 = torch.zeros(1, device=DEV), torch.zeros(1, device=DEV)
    F.dp_clip_factor(t, g, want_norm / 3, work, s2, nrm2, nonfinite=bad)
    assert torch.equal(s2, outs[0][0]) and torch.equal(nrm2, outs[0][1])        # same bits on a second launch
    t[n // 2] = float("nan")
    F.dp_clip_factor(t, g, 1.0, work, s2, nrm2, nonfinite=bad)
    torch.cuda.synchronize()
    assert float(s2) == 0.0 and int(bad) == 1


def _session(arena, wire, dp, **kw):
    from baton_b200.parallel.fedavg import FedAvgSession
    return FedAvgSession(arena, wire_dtype=wire, mode="delta", n_ctas=kw.pop("n_ctas", 8), dp=dp, **kw)


def _drifted_mlp(seed=0, scale=0.01):
    from baton_b200.models import MLP2
    from baton_b200.parallel.arena import ParamArena
    torch.manual_seed(seed)
    m = MLP2(72, 250, 6)
    arena = ParamArena(m, DEV, momentum=True)
    gen = torch.Generator(device=DEV).manual_seed(seed + 1)
    arena.theta.add_(torch.randn(arena.n, device=DEV, generator=gen) * scale)
    return m, arena


@pytest.mark.gpu
@pytest.mark.parametrize("wire", ["fp32", "bf16", "fp8"])
def test_world1_collective_without_noise_applies_the_clipped_update(wire):
    m, arena = _drifted_mlp()
    g0 = arena.global_w.clone()
    delta = (arena.theta - g0).double()
    norm = float(delta.norm())
    sess = _session(arena, wire, DPConfig(norm / 2, 0.0, seed=1))
    assert not sess.use_nvls
    sess.aggregate(my_n=1.0)
    torch.cuda.synchronize()
    sess.check()
    assert sess.last_clip_factors()[0] == pytest.approx(0.5, rel=1e-5)
    want = 0.5 * delta
    got = (arena.global_w.double() - g0.double())
    if wire == "fp32":
        assert float((got - want).abs().max()) < 1e-6
    elif wire == "bf16":
        assert float((got - want).abs().max()) < 3e-4
    else:
        rms = float((got - want).pow(2).mean().sqrt() / want.pow(2).mean().sqrt())
        assert rms < 0.06, rms
    assert torch.equal(arena.theta, arena.global_w)
    assert torch.equal(arena.theta_bf16, arena.theta.to(BF16))
    assert float(arena.momentum.abs().max()) == 0.0


@pytest.mark.gpu
def test_world1_collective_noise_is_the_philox_stream():
    m, arena = _drifted_mlp(seed=3)
    g0 = arena.global_w.clone()
    delta = (arena.theta - g0).double()
    clip = float(delta.norm()) / 4
    dp = DPConfig(clip, 1.5, seed=0xDEADBEEF_12345678)
    sess = _session(arena, "fp32", dp)
    z_dev = []
    for rnd in range(2):
        g_before = arena.global_w.clone().double()
        d = (arena.theta.double() - g_before)
        s = min(1.0, clip / float(d.norm()))
        sess.aggregate(my_n=1.0)
        torch.cuda.synchronize()
        sess.check()
        z = (arena.global_w.double() - g_before - s * d) / dp.noise_std
        want = torch.from_numpy(normals(dp.seed, rnd, arena.n)).to(DEV)
        assert float((z - want).abs().max()) < 1e-4, (rnd, float((z - want).abs().max()))
        z_dev.append(z)
        arena.theta.add_(torch.randn_like(arena.theta) * 0.01)
    assert float((z_dev[0] - z_dev[1]).abs().max()) > 1.0          # a new stream every round


@pytest.mark.gpu
def test_dp_collective_is_invariant_to_ctas_and_tile_size():
    results = []
    for n_ctas in (8, 32, 132):
        for tile in (1024, 4096):
            m, arena = _drifted_mlp(seed=5)
            sess = _session(arena, "fp32", DPConfig(0.05, 1.0, seed=77), n_ctas=n_ctas, tile_elems=tile)
            sess.aggregate(my_n=1.0)
            torch.cuda.synchronize()
            sess.check()
            results.append(arena.global_w.clone())
    for r in results[1:]:
        assert torch.equal(r, results[0])


@pytest.mark.gpu
@pytest.mark.parametrize("wire", ["bf16", "fp32"])
def test_dp_upload_emitted_by_the_optimizer_matches_in_kernel_pack(wire):
    from baton_b200.models import resnet18
    from baton_b200.ops import functional as F
    from baton_b200.parallel.arena import ParamArena
    results = []
    for prepack in (False, True):
        torch.manual_seed(0)
        m = resnet18(10)
        arena = ParamArena(m, DEV)
        sess = _session(arena, wire, DPConfig(0.5, 0.01, seed=11), n_ctas=32)
        hyper = torch.tensor([0.1, 0.0, 0.0, 0.0], device=DEV)
        gen = torch.Generator(device=DEV).manual_seed(7)
        for rnd in range(3):
            arena.grad.copy_(torch.randn(arena.n_param, device=DEV, generator=gen) * 0.01)
            arena.theta[arena.n_param:].add_(0.001 * (rnd + 1))
            if prepack:
                sess.arm_prepack(1.0)
            F.fused_sgd(arena.theta[: arena.n_param], arena.grad, hyper, None, arena.theta_bf16[: arena.n_param],
                        pack=sess.pack_spec() if prepack else None)
            sess.aggregate(my_n=1.0, prepacked=prepack)
            assert sess.last_prepacked == prepack
        torch.cuda.synchronize()
        sess.check()
        assert 0.0 < sess.last_clip_factors()[0] < 1.0
        results.append((arena.theta.clone(), arena.global_w.clone(), arena.theta_bf16.clone()))
    for a, b in zip(*results):
        assert torch.equal(a, b)


@pytest.mark.gpu
def test_engine_logical_clients_equal_the_mean_of_the_clipped_deltas():
    """One GPU hosting 4 logical clients: the clipped fold (norm kernel -> device scalar -> scaled fold, no host read)
    gives the float64 mean of the individually clipped updates of the same clients, each trained alone (full-batch
    steps, so the order of the samples does not matter)."""
    from baton_b200.models import MLP2
    from baton_b200.parallel.engine import FederatedEngine

    def shard(cid):
        gen = torch.Generator().manual_seed(500 + cid)
        X = torch.randn(256, 32, generator=gen)
        return X.to(DEV), (X[:, :4].argmax(1) + cid % 2).clamp_max(3).to(DEV)

    def model():
        torch.manual_seed(0)
        return MLP2(32, 64, 4)
    deltas = []
    for cid in range(4):
        ref = FederatedEngine(model(), DEV, backend="fused", lr=0.1, batch_size=256, wire_dtype="fp32", n_ctas=8)
        g0 = ref.arena.global_w.clone().double()
        ref.run_round(shard(cid), n_epoch=2)
        ref.sync()
        deltas.append(ref.arena.global_w.double() - g0)
    clip = 0.5 * float(torch.stack([d.norm() for d in deltas]).median())
    eng = FederatedEngine(model(), DEV, backend="fused", lr=0.1, batch_size=256, wire_dtype="fp32", n_ctas=8,
                          logical_clients=4, dp_clip=clip, dp_seed=3)
    g0 = eng.arena.global_w.clone().double()
    eng.run_round(shard, n_epoch=2)
    torch.cuda.synchronize()
    s = [min(1.0, clip / float(d.norm())) for d in deltas]
    assert eng.last_clip_factors() == pytest.approx(s, rel=1e-4)
    assert min(s) < 1.0
    want = g0 + sum(si * d for si, d in zip(s, deltas)) / 4
    err = float((eng.arena.global_w.double() - want).abs().max())
    assert err < 1e-5 * max(1.0, float(max(d.abs().max() for d in deltas))), err
    assert math.isinf(eng.privacy_spent(1e-5)[0])          # no noise: no guarantee


@pytest.mark.gpu
def test_k3_engine_dp_round_matches_the_plain_dp_round():
    """bcast_gemm + the optimizer-emitted upload under DP: same seed, same data -> the same clip factor and the same
    global model as the plain DP engine, within the run-to-run spread of two plain runs (training atomics)."""
    from baton_b200.data import ShardSpec, image_shard
    from baton_b200.models import resnet18
    from baton_b200.parallel.engine import FederatedEngine
    X, y = image_shard(ShardSpec(0, torch.full((10,), 0.1), 512), noise=0.3)
    X, y = X.to(DEV).to(BF16), y.to(DEV)
    runs = []
    for k3 in (False, False, True):
        torch.manual_seed(0)
        eng = FederatedEngine(resnet18(10), DEV, backend="fused", lr=0.05, batch_size=128, tile_flags=k3, n_ctas=64,
                              dp_clip=1.0, dp_noise_multiplier=0.01, dp_seed=42)
        assert eng.k3 == k3 and not eng.session.use_nvls
        g0 = eng.arena.global_w.clone()
        factors = []
        for _ in range(2):
            eng.run_round((X, y), n_epoch=1)
            factors += eng.last_clip_factors()
        eng.sync()
        torch.cuda.synchronize()
        eng.session.check()
        if k3:
            assert eng.session.last_prepacked
        assert all(0.0 < s < 1.0 for s in factors), factors          # C = 1 clips this update: the factor matters
        assert math.isfinite(eng.privacy_spent(1e-5)[0])
        runs.append(((eng.arena.global_w - g0).double(), factors))
    (plain_a, s_a), (plain_b, s_b), (k3_d, s_k3) = runs
    spread = float((plain_a - plain_b).norm() / plain_a.norm())
    rel = float((k3_d - plain_a).norm() / plain_a.norm())
    assert rel <= max(3 * spread, 5e-3), (rel, spread)
    for sa, sb, sk in zip(s_a, s_b, s_k3):
        assert abs(sk - sa) <= max(3 * abs(sa - sb), 1e-3 * sa), (s_a, s_b, s_k3)


@pytest.mark.gpu
@pytest.mark.multigpu
def test_fused_dp_collective_multi_gpu_matches_nccl_oracle():
    """At 2..8 GPUs (tests/mp_dp_check.py): the fused DP collective against NcclSession at the same seed over several
    rounds, a rank left out of the alive mask, and a rank whose update is not finite."""
    import os
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    n = min(torch.cuda.device_count(), 8)
    port = 29500 + ((os.getpid() + 541) % 1000)
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(n),
           "--master-addr", "127.0.0.1", "--master-port", str(port), os.path.join(root, "tests", "mp_dp_check.py")]
    proc = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=900, cwd=root)
    tail = "\n".join(proc.stdout.splitlines()[-60:])
    assert proc.returncode == 0 and "RESULT PASS" in proc.stdout, tail
