"""Robust aggregation on the GPU: the robust instantiations of the fused collective against ``robust_combine`` (bitwise
on fp32 and bf16 wires), their invariance to the tiling, the CTA count and the segment order, non-finite clients,
``pack_client`` against the collective's own pack, and engine rounds with logical clients against a host replay."""
import pytest
import torch

from baton_b200.parallel.robust import RobustConfig, robust_combine

BF16 = torch.bfloat16
DEV = "cuda:0"
pytestmark = pytest.mark.gpu


def _bits(t):
    return t.contiguous().view(torch.int32)


def _arena(seed=0):
    from baton_b200.models import MLP2
    from baton_b200.parallel.arena import ParamArena
    torch.manual_seed(seed)
    return ParamArena(MLP2(72, 250, 6), DEV, momentum=True)


def _session(arena, wire, cfg, S, **kw):
    from baton_b200.parallel.fedavg import FedAvgSession
    return FedAvgSession(arena, wire_dtype=wire, mode="delta", n_ctas=kw.pop("n_ctas", 8), robust=cfg, max_clients=S,
                         **kw)


def _deltas(n, S, seed, scale=0.01):
    gen = torch.Generator(device=DEV).manual_seed(seed)
    return [torch.randn(n, device=DEV, generator=gen) * scale * (1 + j % 3) for j in range(S)]


def _round(arena, sess, deltas, order=None):
    """Pack every client's theta = global + d_j into its segment (in ``order``), then run the robust round."""
    g0 = arena.global_w.clone()
    order = list(range(len(deltas))) if order is None else order
    for j, i in enumerate(order):
        arena.theta.copy_(g0 + deltas[i])
        sess.pack_client(j, reset=j + 1 < len(order))
    sess.aggregate(my_n=float(len(deltas)), n_clients=len(deltas))
    torch.cuda.synchronize()
    sess.check()
    return g0


def _wire_decoded(x, wire):
    return x.to(BF16).float() if wire == "bf16" else x.clone()


def _oracle(g0, deltas, cfg, wire):
    stack = torch.stack([_wire_decoded(g0 + d - g0, wire) for d in deltas])
    return g0 + _wire_decoded(robust_combine(stack, cfg), wire)


@pytest.mark.parametrize("wire", ["fp32", "bf16"])
@pytest.mark.parametrize("kind", ["median", "trimmed_mean"])
@pytest.mark.parametrize("S", [1, 2, 7, 8, 32])
def test_world1_kernel_equals_robust_combine(wire, kind, S):
    arena = _arena(S)
    cfg = RobustConfig(kind, 0.2)
    sess = _session(arena, wire, cfg, S)
    assert not sess.use_nvls
    deltas = _deltas(arena.n, S, seed=S)
    g0 = _round(arena, sess, deltas)
    want = _oracle(g0, deltas, cfg, wire)
    assert torch.equal(_bits(arena.global_w), _bits(want))
    assert torch.equal(arena.theta, arena.global_w)
    assert torch.equal(arena.theta_bf16, arena.theta.to(BF16))
    assert float(arena.momentum.abs().max()) == 0.0


@pytest.mark.parametrize("kind", ["median", "trimmed_mean"])
def test_world1_fp8_within_block_scaled_error(kind):
    arena = _arena(3)
    cfg = RobustConfig(kind, 0.25)
    sess = _session(arena, "fp8", cfg, 8)
    deltas = _deltas(arena.n, 8, seed=11)
    g0 = _round(arena, sess, deltas)
    want = robust_combine(torch.stack(deltas), cfg).double()
    got = arena.global_w.double() - g0.double()
    rms = float((got - want).pow(2).mean().sqrt() / want.pow(2).mean().sqrt())
    assert rms < 0.06, rms


@pytest.mark.parametrize("wire", ["fp32", "bf16", "fp8"])
def test_result_is_invariant_to_ctas_tiles_and_segment_order(wire):
    cfg = RobustConfig("trimmed_mean", 0.2)
    results = []
    for n_ctas, tile, order in ((8, 1024, None), (132, 4096, None), (32, 0, [6, 2, 0, 5, 1, 4, 3])):
        arena = _arena(5)
        sess = _session(arena, wire, cfg, 7, n_ctas=n_ctas, tile_elems=tile)
        _round(arena, sess, _deltas(arena.n, 7, seed=21), order=order)
        results.append(arena.global_w.clone())
    for r in results[1:]:
        assert torch.equal(_bits(r), _bits(results[0]))


def test_nonfinite_clients_are_outvoted_by_the_median():
    arena = _arena(7)
    cfg = RobustConfig("median")
    sess = _session(arena, "fp32", cfg, 7)
    deltas = _deltas(arena.n, 7, seed=31)
    deltas[1] = torch.full_like(deltas[1], float("nan"))
    deltas[4] = torch.full_like(deltas[4], float("nan"))
    deltas[5] = torch.full_like(deltas[5], float("inf"))
    g0 = _round(arena, sess, deltas)
    assert bool(torch.isfinite(arena.global_w).all())
    want = g0 + robust_combine(torch.stack(deltas), cfg)     # the 4th value of 4 finite, inf, NaN, NaN
    assert torch.equal(_bits(arena.global_w), _bits(want))
    assert torch.equal(arena.theta, arena.global_w)
    assert torch.equal(arena.theta_bf16, arena.theta.to(BF16))
    assert float(arena.momentum.abs().max()) == 0.0


@pytest.mark.parametrize("wire", ["fp32", "bf16", "fp8"])
def test_pack_client_equals_the_collective_pack(wire):
    cfg = RobustConfig("median")
    outs = []
    for use_pack_client in (False, True):
        arena = _arena(9)
        gen = torch.Generator(device=DEV).manual_seed(2)
        arena.theta.add_(torch.randn(arena.n, device=DEV, generator=gen) * 0.01)
        arena.momentum.fill_(1.0)
        g0, t0 = arena.global_w.clone(), arena.theta.clone()
        sess = _session(arena, wire, cfg, 2)
        if use_pack_client:
            sess.pack_client(1, reset=True)            # a second copy in segment 1 and a reset replica
            torch.cuda.synchronize()
            assert torch.equal(arena.theta, g0) and torch.equal(arena.theta_bf16, g0.to(BF16))
            assert float(arena.momentum.abs().max()) == 0.0
            seg1 = sess.symm.view(sess.off_wire + sess.seg_stride, sess._seg_bytes(arena.n), torch.uint8).clone()
            if wire != "fp8":
                want = (t0 - g0).to(torch.float32 if wire == "fp32" else BF16).view(torch.uint8)
                assert torch.equal(seg1, want)
            arena.theta.copy_(t0)
            sess.pack_client(0)
            seg0 = sess.symm.view(sess.off_wire, sess._seg_bytes(arena.n), torch.uint8)
            assert torch.equal(seg0, seg1)
            sess.aggregate(my_n=1.0, n_clients=1)
        else:
            sess.aggregate(my_n=1.0)                   # the kernel packs seg 0 itself
        torch.cuda.synchronize()
        sess.check()
        outs.append(arena.global_w.clone())
    assert torch.equal(_bits(outs[0]), _bits(outs[1]))


@pytest.mark.parametrize("wire", ["fp32", "bf16"])
def test_optimizer_emitted_upload_gives_the_same_round(wire):
    from baton_b200.ops import functional as F
    cfg = RobustConfig("median")

    def run(prepack):
        arena = _arena(13)
        sess = _session(arena, wire, cfg, 1, nvls=False)
        gen = torch.Generator(device=DEV).manual_seed(7)
        for _ in range(2):
            arena.grad.copy_(torch.randn(arena.n_param, device=DEV, generator=gen) * 0.01)
            if prepack:
                sess.arm_prepack(64.0)
            hyper = torch.tensor([0.1, 0.0, 0.0, 0.0], device=DEV)
            F.fused_sgd(arena.theta[: arena.n_param], arena.grad, hyper, None, arena.theta_bf16[: arena.n_param],
                        pack=sess.pack_spec() if prepack else None)
            sess.aggregate(my_n=64.0, prepacked=prepack)
            assert sess.last_prepacked == prepack
        torch.cuda.synchronize()
        sess.check()
        return arena.global_w.clone()

    assert torch.equal(_bits(run(False)), _bits(run(True)))


def _mlp_engine(aggregator, wire="fp32", **kw):
    from baton_b200.models import MLP2
    from baton_b200.parallel.engine import FederatedEngine
    torch.manual_seed(0)
    return FederatedEngine(MLP2(16, 64, 1), DEV, backend="fused", loss="mse", lr=0.002, batch_size=256,
                           wire_dtype=wire, logical_clients=16, sample_k=8, seed=3, aggregator=aggregator, **kw)


def _shards(n_clients=16):
    """Full-batch shards (256 samples, batch 256): a client's update does not depend on the sample order, so a replay
    that draws its shuffles from another point of the random stream trains the same update."""
    gen = torch.Generator().manual_seed(1)
    data = {}
    for cid in range(n_clients):
        X = torch.randn(256, 16, generator=gen)
        data[cid] = (X.to(DEV), (X @ (torch.arange(1.0, 17.0) * (1 + 0.5 * cid))).unsqueeze(1).to(DEV))
    return data


@pytest.mark.parametrize("aggregator", ["median", "trimmed_mean"])
def test_engine_logical_clients_match_a_host_replay(aggregator):
    """16 logical clients, 8 per round, 3 rounds: the engine's global model matches replaying the same clients with
    the same trainer in a second engine, one at a time from the round's global model, and combining their fp32 deltas
    with robust_combine.  Not bitwise: the two engines' local training agrees in most elements but not in every last
    bit, and a last-bit change in one client's delta can change which client an element's statistic selects.  Each
    round is therefore compared by the relative L2 norm of the update difference, bounded by 1e-5 (measured on an
    H100: about 3e-7, with 6 to 9 % of the elements differing in their last bits)."""
    data = _shards()
    eng = _mlp_engine(aggregator, trim_ratio=0.25)
    assert eng.session.max_clients == 8
    ref = _mlp_engine("mean")                           # a second replica only for its trainer
    cfg = RobustConfig(aggregator, 0.25)
    a2 = ref.arena
    for r in range(3):
        g0 = eng.arena.global_w.clone()
        # replay first (the draw uses the engine's rng state: peek by copying it)
        state = eng._rng.getstate()
        parts = eng.draw_participants()
        eng._rng.setstate(state)
        deltas = []
        for cid in parts:
            a2.theta.copy_(g0)
            a2.global_w.copy_(g0)
            a2.sync_shadow()
            if a2.momentum is not None:
                a2.momentum.zero_()
            X, y = data[cid]
            ref.trainer.run(X, y, n_epoch=1, return_device=True, **ref.hp)
            torch.cuda.synchronize()
            deltas.append(a2.theta - g0)
        want = g0 + robust_combine(torch.stack(deltas), cfg)
        res = eng.run_round(lambda c: data[c], n_epoch=1)
        eng.sync()
        torch.cuda.synchronize()
        eng.session.check()
        assert res.participants == parts
        upd, want_upd = eng.arena.global_w - g0, want - g0
        rel = float((upd - want_upd).norm() / want_upd.norm())
        print("round", r, "relative L2 difference of the update", rel, "elements differing",
              int((upd != want_upd).sum()), "of", upd.numel())
        assert rel < 1e-5, (r, rel)


def test_engine_mean_aggregator_is_the_plain_engine():
    from baton_b200.models import MLP2
    from baton_b200.parallel.engine import FederatedEngine
    data = _shards()
    outs = []
    for kw in ({}, {"aggregator": "mean"}):
        torch.manual_seed(0)
        eng = FederatedEngine(MLP2(16, 64, 1), DEV, backend="fused", loss="mse", lr=0.002, batch_size=256,
                              logical_clients=16, sample_k=8, seed=3, **kw)
        for _ in range(3):
            eng.run_round(lambda c: data[c], n_epoch=1)
        eng.sync()
        torch.cuda.synchronize()
        outs.append(eng.arena.global_w.clone())
    assert torch.equal(_bits(outs[0]), _bits(outs[1]))


def test_engine_resnet18_median_round_is_finite_and_moves():
    from baton_b200.data import ShardSpec, image_shard
    from baton_b200.models import resnet18
    from baton_b200.parallel.engine import FederatedEngine
    torch.manual_seed(0)
    eng = FederatedEngine(resnet18(10), DEV, backend="fused", lr=0.05, batch_size=64, logical_clients=4, sample_k=4,
                          aggregator="median")
    assert eng.session.max_clients == 4
    data = {}
    for c in range(4):
        X, y = image_shard(ShardSpec(c, torch.full((10,), 0.1), 128), noise=0.3)
        data[c] = (X.to(DEV).to(BF16), y.to(DEV))
    g0 = eng.arena.global_w.clone()
    eng.run_round(lambda c: data[c], n_epoch=1)
    eng.sync()
    torch.cuda.synchronize()
    eng.session.check()
    assert bool(torch.isfinite(eng.arena.global_w).all())
    assert float((eng.arena.global_w - g0).abs().max()) > 0.0
