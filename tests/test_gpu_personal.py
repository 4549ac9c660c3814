"""Personalized rounds on the GPU (FedBN / FedPer, parallel/personal.py): the LocalArgs collective against the plain
kernel on the compacted arena, bit for bit; ResNet-18 engine rounds with one client per GPU and with logical clients
checked against snapshots of the trained replicas; personalized evaluation; and the multi-GPU check
(tests/mp_personal_check.py, two or more GPUs)."""
import os
import subprocess
import sys

import pytest
import torch
from torch import nn

from baton_b200.parallel.arena import ParamArena
from baton_b200.parallel.personal import resolve_local_keys
from baton_b200.parallel.server_opt import ServerOptConfig

DEV = "cuda:0"
pytestmark = pytest.mark.gpu
BUFS = ("theta", "global_w", "theta_bf16", "momentum")


def _bits(t):
    return t.contiguous().view(torch.int16 if t.dtype == torch.bfloat16 else torch.int32)


def _cut(x, lo, hi):
    return torch.cat((x[:lo], x[hi:]))


class _Compact(nn.Module):
    """Its arena IS the logical vector of a personalized arena: one parameter of lo elements, one buffer of n - hi."""

    def __init__(self, n_lo, n_tail):
        super().__init__()
        self.p = nn.Parameter(torch.zeros(n_lo))
        self.register_buffer("b", torch.zeros(n_tail))


def _session(arena, wire, mode, sopt, local):
    from baton_b200.parallel.fedavg import FedAvgSession
    cfg = ServerOptConfig(sopt, 0.05) if sopt else None
    return FedAvgSession(arena, wire_dtype=wire, mode=mode, n_ctas=16, nvls=False, server_opt=cfg, local=local)


@pytest.mark.parametrize("wire", ["fp32", "bf16", "fp8"])
@pytest.mark.parametrize("mode, sopt", [("delta", None), ("weights", None), ("delta", "avgm"), ("delta", "adam")])
@pytest.mark.parametrize("local_keys", ["bn", "head"])
def test_local_collective_equals_the_plain_kernel_on_the_compacted_arena(wire, mode, sopt, local_keys):
    from baton_b200.models import resnet18
    torch.manual_seed(0)
    m = resnet18(10)
    a = ParamArena(m, DEV, momentum=True, local=resolve_local_keys(m, local_keys))
    lo, hi = a.local_range
    c = ParamArena(_Compact(lo, a.n - hi), DEV, momentum=True, total_align=1024)
    assert c.n == a.n_shared and c.n_param == lo
    s, sc = _session(a, wire, mode, sopt, True), _session(c, wire, mode, sopt, False)
    gen = torch.Generator(device=DEV).manual_seed(11)
    for r in range(2):
        a.global_w.copy_(torch.randn(a.n, device=DEV, generator=gen))
        a.theta.copy_(a.global_w + 0.01 * torch.randn(a.n, device=DEV, generator=gen))
        a.theta_bf16.copy_(torch.randn(a.n, device=DEV, generator=gen))
        a.momentum.fill_(3.0)
        for k in ("theta", "global_w"):
            getattr(c, k).copy_(_cut(getattr(a, k), lo, hi))
        c.theta_bf16.copy_(_cut(a.theta_bf16, lo, hi))
        c.momentum.fill_(3.0)
        before = {k: getattr(a, k).clone() for k in BUFS}
        st0 = [t.clone() for t in (a.server_m, a.server_v) if t is not None]
        s.aggregate(my_n=5.0)
        sc.aggregate(my_n=5.0)
        torch.cuda.synchronize()
        for k in ("theta", "global_w", "theta_bf16"):
            x = getattr(a, k)
            assert torch.equal(_bits(_cut(x, lo, hi)), _bits(getattr(c, k))), (r, k)
        assert torch.equal(a.momentum[:lo], c.momentum), r
        for k in BUFS:       # the local range is never touched, in any buffer
            assert torch.equal(_bits(getattr(a, k)[lo:hi]), _bits(before[k][lo:hi])), (r, k)
        if sopt:
            for x, y, x0 in zip((a.server_m, a.server_v), (c.server_m, c.server_v), st0):
                assert torch.equal(_bits(x[:lo]), _bits(y)) and torch.equal(x[lo:], x0[lo:]), r
    assert s.wire_bytes() == sc.wire_bytes()


def _resnet_engine(local_keys, **kw):
    from baton_b200.models import resnet18
    from baton_b200.parallel.engine import FederatedEngine
    torch.manual_seed(0)
    return FederatedEngine(resnet18(10), DEV, lr=0.05, batch_size=32, momentum=0.9, wire_dtype="fp32", nvls=False,
                           local_keys=local_keys, **kw)


def _shard(cid, n=64):
    from baton_b200.data import dirichlet_label_shards, image_shard
    spec = dirichlet_label_shards(8, 10, n, alpha=0.5, seed=1)[cid]
    X, y = image_shard(spec, shift=0.3)
    return X.to(DEV, torch.bfloat16), y.to(DEV)


@pytest.mark.parametrize("local_keys", ["bn", "head"])
def test_engine_one_client_per_gpu_keeps_its_local_entries(local_keys):
    eng = _resnet_engine(local_keys)
    a = eng.arena
    lo, hi = a.local_range
    snap = {}
    agg = eng.session.aggregate

    def spy(*args, **kw):
        torch.cuda.current_stream().synchronize()
        snap["trained"], snap["global"] = a.theta.clone(), a.global_w.clone()
        return agg(*args, **kw)

    eng.session.aggregate = spy
    X, y = _shard(0)
    for r in range(3):                 # the captured epoch graph is replayed from round 2 on
        start_local = a.theta[lo:hi].clone()
        eng.run_round((X, y), n_epoch=1)
        eng.sync()
        torch.cuda.synchronize()
        t, g = snap["trained"], snap["global"]
        assert torch.equal(snap["global"][lo:hi], start_local), r       # FedProx's anchor: the client's own values
        want = g + (t - g)
        assert torch.equal(_bits(_cut(a.global_w, lo, hi)), _bits(_cut(want, lo, hi))), r
        assert torch.equal(_bits(_cut(a.theta, lo, hi)), _bits(_cut(want, lo, hi))), r
        assert torch.equal(_bits(a.theta[lo:hi]), _bits(t[lo:hi])), r
        got = torch.cat([v.flatten() for v in eng.local_entries(0).values()])
        flat = torch.cat([a._view(t, a.slots[k]).flatten() for k in eng.personal.keys])
        assert torch.equal(got, flat), r
        assert not torch.equal(t[lo:hi], start_local), r                 # the local entries did train


def test_engine_logical_clients_store_and_fold():
    eng = _resnet_engine("bn", logical_clients=4, sample_k=2, seed=3)
    a = eng.arena
    lo, hi = a.local_range
    init = a.theta[lo:hi].clone()
    start, trained = {}, {}
    train = eng._train_client

    def spy(cid, X, y, n_epoch, first):
        start[cid] = a.theta.clone()
        out = train(cid, X, y, n_epoch, first)
        torch.cuda.current_stream().synchronize()
        trained[cid] = a.theta.clone()
        return out

    eng._train_client = spy
    last = {c: init.clone() for c in range(4)}
    for r in range(3):
        g0 = a.global_w.clone()
        start.clear()
        trained.clear()
        res = eng.run_round(_shard, n_epoch=1)
        eng.sync()
        torch.cuda.synchronize()
        parts = res.participants
        for c in range(4):
            if c in parts:
                assert torch.equal(start[c][lo:hi], last[c]), (r, c)
                assert torch.equal(_cut(start[c], lo, hi), _cut(g0, lo, hi)), (r, c)
                last[c] = trained[c][lo:hi].clone()
            got = torch.cat([v.flatten() for v in eng.local_entries(c).values()])
            flat = torch.cat([a._view(torch.cat((torch.zeros(lo, device=DEV), last[c])), a.slots[k]).flatten()
                              for k in eng.personal.keys])
            assert torch.equal(got, flat), (r, c)
        n = {c: float(_shard(c)[0].shape[0]) for c in parts}
        want = g0 + sum(n[c] * (trained[c] - g0) for c in parts) / sum(n.values())
        err = float((_cut(a.global_w, lo, hi) - _cut(want, lo, hi)).abs().max())
        assert err < 1e-6, (r, err)


def _plain_eval(sd, X, y):
    """Eval-mode forward of a fresh copy of the model loaded with ``sd``: (loss sum, #correct)."""
    from baton_b200.models import resnet18
    m = resnet18(10)
    arena = ParamArena(m, DEV)
    m.build_workspace(torch.device(DEV))
    m.load_state_dict(sd)
    arena.commit_global()
    m.eval()
    with torch.no_grad():
        logits = m(X).float()
    return float(nn.functional.cross_entropy(logits, y, reduction="sum")), float((logits.argmax(-1) == y).sum())


def test_evaluate_uses_each_clients_personalized_model():
    eng = _resnet_engine(("bn", "head"), logical_clients=3, sample_k=2, seed=5)
    eng.run_round(_shard, n_epoch=1)
    eng.run_round(_shard, n_epoch=1)
    eng.sync()
    torch.cuda.synchronize()
    a = eng.arena
    before = {k: getattr(a, k).clone() for k in BUFS}
    store = {c: v.clone() for c, v in eng.personal.clients.items()}
    held = {c: _shard(c, 96) for c in range(3)}
    res = eng.evaluate(lambda c: held[c])
    torch.cuda.synchronize()
    for k in BUFS:
        assert torch.equal(_bits(getattr(a, k)), _bits(before[k])), k
    assert set(eng.personal.clients) == set(store) and all(torch.equal(store[c], eng.personal.clients[c]) for c in store)
    tot_loss = tot_correct = 0.0
    for c in range(3):
        one = eng.evaluate(lambda cid, c=c: held[c] if cid == c else None)
        ls, cr = _plain_eval(eng.client_state_dict(c), *held[c])
        assert abs(one.local_loss * one.local_n_samples - ls) <= 2e-2 * abs(ls) + 1e-2, c
        assert abs(one.local_accuracy * one.local_n_samples - cr) <= 2, c
        tot_loss += ls
        tot_correct += cr
    assert abs(res.loss * res.n_samples - tot_loss) <= 2e-2 * abs(tot_loss) + 1e-2
    for k in BUFS:
        assert torch.equal(_bits(getattr(a, k)), _bits(before[k])), k


def test_multi_gpu_shared_agree_and_local_differ():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 or more GPUs")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    port = 29400 + ((os.getpid() + 409) % 500)
    n = min(torch.cuda.device_count(), 8)
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(n),
           "--master-addr", "127.0.0.1", "--master-port", str(port), os.path.join(root, "tests", "mp_personal_check.py")]
    proc = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=900, cwd=root)
    tail = "\n".join(proc.stdout.splitlines()[-40:])
    assert proc.returncode == 0 and "RESULT PASS" in proc.stdout, tail
