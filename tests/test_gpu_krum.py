"""Multi-Krum on the GPU: the Krum instantiations of the fused collective against the host oracle (the kept set, the
global model bitwise on fp32 and bf16 wires, the distances to 1e-5), fp8 within the block-scaled error, invariance to
the CTA count, the tiling and the segment order, scaled / sign-flipped / NaN attackers, engine rounds with logical
clients against a host replay, and (with >= 2 GPUs) the multi-rank collective against ``NcclSession``."""
import os
import subprocess
import sys

import pytest
import torch

from baton_b200.parallel.robust import RobustConfig, krum_select, robust_combine

BF16 = torch.bfloat16
DEV = "cuda:0"
pytestmark = pytest.mark.gpu
MEAN = RobustConfig("trimmed_mean", 0.0)


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


def _deltas(n, S, seed):
    """Well-separated clients: a shared direction plus client noise whose size grows with the client index, so every
    score differs from the others by far more than the device's rounding."""
    gen = torch.Generator(device=DEV).manual_seed(seed)
    common = torch.randn(n, device=DEV, generator=gen) * 0.01
    return [common + torch.randn(n, device=DEV, generator=gen) * 0.004 * (1 + 0.45 * j) for j in range(S)]


def _round(arena, sess, deltas, order=None):
    g0 = arena.global_w.clone()
    order = list(range(len(deltas))) if order is None else order
    for j, i in enumerate(order):
        arena.theta.copy_(g0 + deltas[i])
        sess.pack_client(j, reset=j + 1 < len(order))
    sess.aggregate(my_n=float(len(deltas)), n_clients=len(deltas))
    torch.cuda.synchronize()
    sess.check()
    return g0


def _decoded(x, wire):
    return x.to(BF16).float() if wire == "bf16" else x.clone()


def _f(S):
    return min(max((S - 3) // 2, 0), 4)


@pytest.mark.parametrize("wire", ["fp32", "bf16"])
@pytest.mark.parametrize("S", [1, 2, 3, 7, 8, 16, 32])
def test_world1_kernel_equals_the_oracle(wire, S):
    arena = _arena(S)
    cfg = RobustConfig("krum", krum_f=_f(S))
    sess = _session(arena, wire, cfg, S)
    assert not sess.use_nvls and sess.krum
    deltas = _deltas(arena.n, S, seed=S)
    g0 = _round(arena, sess, deltas)
    stack = torch.stack([_decoded(g0 + d - g0, wire) for d in deltas])       # what pack_client uploads
    D, scores, kept = krum_select(stack, cfg)
    dD, dscores, dkept = sess.last_krum()
    assert dkept.tolist() == kept.tolist()
    assert int(kept.sum()) == cfg.krum_kept(S)
    if S >= 3:                       # P <= 2 skips the distances: every score ties
        off = ~torch.eye(S, dtype=torch.bool)
        rel = float(((dD - D).abs()[off] / D[off]).max())
        assert rel < 1e-5, rel
        assert float(((dscores - scores).abs() / scores).max()) < 1e-5
    want = g0 + _decoded(robust_combine(stack[kept.to(DEV)], MEAN), wire)
    assert torch.equal(_bits(arena.global_w), _bits(want))
    assert torch.equal(arena.theta, arena.global_w)
    assert torch.equal(arena.theta_bf16, arena.theta.to(BF16))
    assert float(arena.momentum.abs().max()) == 0.0


def test_world1_fp8_within_block_scaled_error():
    arena = _arena(3)
    cfg = RobustConfig("krum", krum_f=2)
    sess = _session(arena, "fp8", cfg, 8)
    deltas = _deltas(arena.n, 8, seed=11)
    g0 = _round(arena, sess, deltas)
    kept = krum_select(torch.stack(deltas), cfg)[2]
    assert sess.last_krum()[2].tolist() == kept.tolist()
    want = robust_combine(torch.stack(deltas), cfg).double()
    got = arena.global_w.double() - g0.double()
    rms = float((got - want).pow(2).mean().sqrt() / want.pow(2).mean().sqrt())
    assert rms < 0.06, rms


@pytest.mark.parametrize("wire", ["fp32", "bf16", "fp8"])
def test_result_is_invariant_to_ctas_tiles_and_segment_order(wire):
    cfg = RobustConfig("krum", krum_f=2)
    results, kept_ids = [], []
    for n_ctas, tile, order in ((8, 1024, None), (132, 4096, None), (32, 0, [6, 2, 0, 5, 1, 4, 3])):
        arena = _arena(5)
        sess = _session(arena, wire, cfg, 7, n_ctas=n_ctas, tile_elems=tile)
        _round(arena, sess, _deltas(arena.n, 7, seed=21), order=order)
        kept = sess.last_krum()[2].tolist()
        pos = order or list(range(7))
        kept_ids.append(sorted(pos[j] for j in range(7) if kept[j]))
        results.append(arena.global_w.clone())
    assert kept_ids[1] == kept_ids[0] and kept_ids[2] == kept_ids[0]
    for r in results[1:]:
        assert torch.equal(_bits(r), _bits(results[0]))


@pytest.mark.parametrize("attack", ["scaled", "sign_flipped", "nan"])
def test_attackers_are_never_kept(attack):
    arena = _arena(7)
    cfg = RobustConfig("krum", krum_f=2)
    sess = _session(arena, "bf16", cfg, 8)
    deltas = _deltas(arena.n, 8, seed=31)
    for j in (1, 6):
        deltas[j] = {"scaled": deltas[j] * 100.0, "sign_flipped": deltas[j] * -10.0,
                     "nan": torch.full_like(deltas[j], float("nan"))}[attack]
    g0 = _round(arena, sess, deltas)
    kept = sess.last_krum()[2].tolist()
    assert not kept[1] and not kept[6] and sum(kept) == 6
    assert bool(torch.isfinite(arena.global_w).all())
    stack = torch.stack([_decoded(g0 + d - g0, "bf16") for d in deltas])
    want = g0 + _decoded(robust_combine(stack, cfg), "bf16")
    assert torch.equal(_bits(arena.global_w), _bits(want))


def test_krum_round_needs_a_krum_session():
    arena = _arena(2)
    sess = _session(arena, "fp32", RobustConfig("median"), 2)
    with pytest.raises(ValueError):
        sess.aggregate(my_n=1.0, robust=RobustConfig("krum"))
    with pytest.raises(RuntimeError):
        sess.last_krum()


def _mlp_engine(aggregator, **kw):
    from baton_b200.models import MLP2
    from baton_b200.parallel.engine import FederatedEngine
    torch.manual_seed(0)
    return FederatedEngine(MLP2(16, 64, 1), DEV, backend="fused", loss="mse", lr=0.002, batch_size=256,
                           wire_dtype="fp32", logical_clients=16, sample_k=8, seed=3, aggregator=aggregator, **kw)


def _shards(n_clients=16):
    """Full-batch shards: a client's update does not depend on the sample order, so a replay trains the same update."""
    gen = torch.Generator().manual_seed(1)
    data = {}
    for cid in range(n_clients):
        X = torch.randn(256, 16, generator=gen)
        sign = -4.0 if cid in (3, 11) else 1.0
        data[cid] = (X.to(DEV), (X @ (torch.arange(1.0, 17.0) * (1 + 0.5 * cid) * sign)).unsqueeze(1).to(DEV))
    return data


def test_engine_logical_clients_match_a_host_replay():
    """16 logical clients, 8 per round, 3 rounds: the engine's kept set equals the oracle's over the same clients
    replayed one at a time from the round's global model, and its update matches theirs to 1e-5 relative L2 (the two
    engines' local training agrees to the last bits in most, not all, elements); last_krum names the clients."""
    data = _shards()
    eng = _mlp_engine("krum", krum_f=2)
    assert eng.session.max_clients == 8
    ref = _mlp_engine("mean")
    cfg = RobustConfig("krum", krum_f=2)
    a2 = ref.arena
    for r in range(3):
        g0 = eng.arena.global_w.clone()
        state = eng._rng.getstate()
        parts = eng.draw_participants()
        eng._rng.setstate(state)
        order = list(parts)                            # world 1: segment order is the draw order
        deltas = []
        for cid in order:
            a2.theta.copy_(g0)
            a2.global_w.copy_(g0)
            a2.sync_shadow()
            X, y = data[cid]
            ref.trainer.run(X, y, n_epoch=1, return_device=True, **ref.hp)
            torch.cuda.synchronize()
            deltas.append(a2.theta - g0)
        stack = torch.stack(deltas)
        _, scores, kept = krum_select(stack, cfg)
        want = g0 + robust_combine(stack, cfg)
        res = eng.run_round(lambda c: data[c], n_epoch=1)
        eng.sync()
        torch.cuda.synchronize()
        eng.session.check()
        assert res.participants == parts
        rep = eng.last_krum()
        assert sorted(rep) == sorted(parts)
        assert [rep[c][1] for c in order] == kept.tolist()
        assert not any(rep[c][1] for c in (3, 11) if c in rep)
        upd, want_upd = eng.arena.global_w - g0, want - g0
        rel = float((upd - want_upd).norm() / want_upd.norm())
        print("round", r, "kept", [c for c in order if rep[c][1]], "relative L2 difference", rel)
        assert rel < 1e-5, (r, rel)


@pytest.mark.multigpu
def test_fused_krum_collective_multi_gpu_matches_nccl_oracle():
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    n = min(torch.cuda.device_count(), 8)
    port = 29500 + ((os.getpid() + 739) % 1000)
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(n),
           "--master-addr", "127.0.0.1", "--master-port", str(port), os.path.join(root, "tests", "mp_krum_check.py")]
    proc = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=900, cwd=root)
    tail = "\n".join(proc.stdout.splitlines()[-60:])
    assert proc.returncode == 0 and "RESULT PASS" in proc.stdout, tail
