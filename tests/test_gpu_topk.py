"""Top-k uploads with error feedback on the GPU: the selection and compaction kernels against the host rule
(parallel/compress.py) bit for bit, the sparse collective against topk_combine, the ratio-1 identity with the plain
session for one client and for folded logical clients (with and without FedAdam), and ResNet-18 engine rounds against
backend='nccl'."""
import os
import subprocess
import sys

import pytest
import torch

from baton_b200.parallel.compress import (GRANULE, TopKConfig, n_float, sparse_upload_bytes, topk_combine, topk_ef_,
                                          topk_select)
from baton_b200.parallel.server_opt import ServerOptConfig

DEV = "cuda:0"
pytestmark = pytest.mark.gpu
RESNET18_N = 11_190_272          # ResNet-18 (10 classes) float elements rounded up to whole granules


def _bits(t):
    return t.contiguous().view(torch.int32)


def _same(a, b):
    """Bitwise equal, every NaN counting as one value."""
    na, nb = torch.isnan(a), torch.isnan(b)
    return torch.equal(na, nb) and torch.equal(_bits(a[~na]), _bits(b[~nb]))


def _lists(n, cap, wire):
    vdt = torch.float32 if wire == "fp32" else torch.bfloat16
    return (torch.zeros(n // GRANULE + 1, dtype=torch.int32, device=DEV), torch.zeros(cap, dtype=torch.int16, device=DEV),
            torch.zeros(cap, dtype=vdt, device=DEV))


def _entries(rowptr, off, val):
    """Arena indices and fp32 values of a sparse list (host)."""
    rp = rowptr.cpu().long()
    cnt = rp[1:] - rp[:-1]
    m = int(rp[-1])
    gran = torch.repeat_interleave(torch.arange(cnt.numel()), cnt)
    idx = gran * GRANULE + (off[:m].cpu().long() & 0xFFFF)
    return idx, val[:m].float().cpu()


def _pack(theta, g, e, k, wire, ef=True, cap=None):
    from baton_b200.ops import functional as F
    n = theta.numel()
    cap = cap or k
    rowptr, off, val = _lists(n, cap, wire)
    u = e if ef else torch.empty_like(theta)
    F.topk_pack(theta, g, u, k, F.topk_work(n, DEV), rowptr.data_ptr(), off.data_ptr(), val.data_ptr(), ef=ef,
                wire_fp32=wire == "fp32", cap=cap)
    torch.cuda.synchronize()
    return rowptr, off, val


def _inputs(kind, n, seed):
    gen = torch.Generator(device=DEV).manual_seed(seed)
    g = torch.randn(n, device=DEV, generator=gen)
    d = torch.randn(n, device=DEV, generator=gen) * 1e-3
    if kind == "tied":
        d = torch.round(d * 2e3) / 2e3          # a handful of magnitudes: long runs of ties at the threshold
    elif kind == "special":
        d[::97] = float("nan")
        d[5::1013] = float("inf")
        d[7::1013] = -float("inf")
        d[9::331] = 0.0
        d[11::331] = -0.0
    elif kind == "zero":
        d.zero_()
    e = torch.randn(n, device=DEV, generator=gen) * 1e-4 if kind != "zero" else torch.zeros(n, device=DEV)
    return g + d, g, e


@pytest.mark.parametrize("kind,n,ratio", [("random", 1 << 20, 0.01), ("tied", 1 << 20, 0.05), ("special", 1 << 18, 0.1),
                                          ("zero", 1 << 16, 0.01), ("random", RESNET18_N, 0.01),
                                          ("tied", RESNET18_N, 0.001)])
@pytest.mark.parametrize("wire", ["fp32", "bf16"])
def test_selection_matches_the_host_rule(kind, n, ratio, wire):
    theta, g, e = _inputs(kind, n, seed=n % 97)
    k = TopKConfig(ratio).k(n)
    e_host = e.clone()
    idx_h, vals_h = topk_ef_(theta, g, e_host, k)
    e1 = e.clone()
    rowptr, off, val = _pack(theta, g, e1, k, wire)
    idx, vals = _entries(rowptr, off, val)
    assert int(rowptr[-1]) == k
    assert torch.equal(idx, idx_h.cpu())
    want = vals_h.float().cpu() if wire == "fp32" else vals_h.to(torch.bfloat16).float().cpu()
    assert _same(vals, want)
    assert _same(e1, e_host)
    # a second launch on the same inputs gives the same bits
    e2 = e.clone()
    r2, o2, v2 = _pack(theta, g, e2, k, wire)
    assert torch.equal(r2, rowptr) and torch.equal(o2, off) and _same(v2.float(), val.float())
    assert _same(e2, e1)


@pytest.mark.parametrize("k", [1, 3, 1 << 16])
def test_selection_edge_sizes_and_no_error_feedback(k):
    n = 1 << 16
    theta, g, e = _inputs("tied", n, seed=k)
    rowptr, off, val = _pack(theta, g, e, k, "fp32", ef=False)
    idx, vals = _entries(rowptr, off, val)
    u = theta - g
    assert torch.equal(idx, topk_select(u, k).cpu())
    assert torch.equal(_bits(vals), _bits(u[idx.to(DEV)].cpu()))


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


def _session(arena, wire, **kw):
    from baton_b200.parallel.fedavg import FedAvgSession
    return FedAvgSession(arena, wire_dtype=wire, mode="delta", n_ctas=kw.pop("n_ctas", 8), nvls=False, **kw)


def _delta(arena, seed, scale=0.01):
    gen = torch.Generator(device=DEV).manual_seed(seed)
    d = torch.randn(arena.n, device=DEV, generator=gen) * scale
    mask = torch.zeros(arena.n, device=DEV)
    for s in arena.slots.values():          # the alignment padding stays at the global model, as in training
        mask[s.offset: s.offset + s.numel] = 1.0
    return d * mask


@pytest.mark.parametrize("wire", ["fp32", "bf16"])
@pytest.mark.parametrize("sopt", [None, "adam"])
def test_world1_collective_equals_topk_combine(wire, sopt):
    cfg = ServerOptConfig(sopt, lr=0.01) if sopt else None
    a = _arena()
    s = _session(a, wire, topk=TopKConfig(0.05), server_opt=cfg)
    e = torch.zeros(a.n, device=DEV)
    x = a.global_w.clone()
    for r in range(3):
        a.theta.copy_(a.global_w + _delta(a, 10 + r))
        e_host = e.clone()
        idx, vals = topk_ef_(a.theta, a.global_w, e_host, s.topk_k)
        s.pack_topk(e)
        s.aggregate(my_n=5.0)
        torch.cuda.synchronize()
        s.check()
        assert s.last_upload_entries() == s.topk_k == idx.numel()
        assert s.last_upload_bytes() == sparse_upload_bytes(a.n, s.topk_k, wire)
        vw = vals.float() if wire == "fp32" else vals.to(torch.bfloat16)
        d = topk_combine([(idx, vw)], [1.0], a.n, wire).to(DEV)
        if cfg is None:
            x = x + d
        else:
            from baton_b200.parallel.server_opt import apply_update_
            if r == 0:
                m, v = cfg.init_state(a.n_param, DEV)
            apply_update_(x, d, a.n_param, m, v, cfg)
        assert torch.equal(_bits(e), _bits(e_host))
        assert torch.equal(_bits(a.global_w), _bits(x)) and torch.equal(a.theta, a.global_w)


def _identity_rounds(wire, n_clients, sopt, rounds=2):
    """The same client updates through a plain session and a ratio-1 top-k session: global models per round."""
    from baton_b200.ops import functional as F
    cfg = ServerOptConfig(sopt, lr=0.01) if sopt else None
    out = []
    for topk in (None, TopKConfig(1.0)):
        a = _arena()
        kw = {"topk": topk, "max_clients": n_clients} if topk else {}
        s = _session(a, wire, server_opt=cfg, **kw)
        acc = torch.zeros_like(a.theta)
        res = {j: torch.zeros(a.n, device=DEV) for j in range(n_clients)}
        hist = []
        for r in range(rounds):
            total = 0.0
            for j in range(n_clients):
                a.theta.copy_(a.global_w + _delta(a, 100 * r + j))
                nk = float(3 + j)
                total += nk
                if n_clients == 1:
                    if topk:
                        s.pack_topk(res[j])
                elif topk:
                    s.fold_topk(acc, res[j], nk, first=j == 0, reset=j + 1 < n_clients)
                else:
                    F.fold_client(acc, a.theta, a.global_w, nk, first=j == 0, reset=j + 1 < n_clients,
                                  w_bf16=a.theta_bf16, momentum=a.momentum)
            if n_clients > 1:
                F.fold_finish(acc, a.theta, a.global_w, total)
                if topk:
                    s.pack_nonzero()
            s.aggregate(my_n=total)
            torch.cuda.synchronize()
            s.check()
            hist.append(a.global_w.clone())
            if topk:
                assert all(int(torch.count_nonzero(e)) == 0 for e in res.values())
        out.append(hist)
    return out


@pytest.mark.parametrize("wire", ["fp32", "bf16"])
@pytest.mark.parametrize("n_clients", [1, 4])
@pytest.mark.parametrize("sopt", [None, "adam"])
def test_ratio_one_is_the_plain_round_bit_for_bit(wire, n_clients, sopt):
    plain, topk = _identity_rounds(wire, n_clients, sopt)
    for p, t in zip(plain, topk):
        assert torch.equal(_bits(p), _bits(t))


def test_fold_of_one_client_equals_its_own_upload():
    """A single hosted client's list (pack_topk) and the same client folded alone (fold_topk + fold_finish +
    pack_nonzero) give the same round on an fp32 wire."""
    from baton_b200.ops import functional as F
    res = []
    for fold in (False, True):
        a = _arena()
        s = _session(a, "fp32", topk=TopKConfig(0.02))
        e = torch.zeros(a.n, device=DEV)
        a.theta.copy_(a.global_w + _delta(a, 7))
        if fold:
            acc = torch.zeros_like(a.theta)
            s.fold_topk(acc, e, 4.0, first=True, reset=False)
            F.fold_finish(acc, a.theta, a.global_w, 4.0)
            s.pack_nonzero()
        else:
            s.pack_topk(e)
        s.aggregate(my_n=4.0)
        torch.cuda.synchronize()
        res.append((a.global_w.clone(), e.clone(), s.last_upload_entries()))
    (g0, e0, k0), (g1, e1, k1) = res
    assert torch.equal(e0, e1) and k1 <= k0
    assert torch.allclose(g0, g1, rtol=1e-6, atol=1e-9)   # fold_finish rounds n_k * x / n_k once more


def _rel(a, b):
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


def test_resnet18_engine_topk_logical_clients_fused_matches_nccl():
    """Three rounds of ResNet-18, 8 logical clients with 4 sampled, top-k 1 % with error feedback: backend='fused'
    against backend='nccl' (the difference calibrated by two fused runs: training accumulates BatchNorm statistics with
    fp32 atomics, so runs differ in the last bits and the selection can differ at its margin)."""
    from baton_b200.models import resnet18
    from baton_b200.parallel.engine import FederatedEngine
    from test_gpu_fedprox import _image_data
    X, y = _image_data(DEV, 512)
    shards = lambda c: (X[64 * c: 64 * c + 64], y[64 * c: 64 * c + 64])    # noqa: E731

    def run(backend):
        torch.manual_seed(0)
        eng = FederatedEngine(resnet18(10), DEV, backend=backend, lr=0.05, batch_size=32, n_ctas=64,
                              logical_clients=8, sample_k=4, compress="topk", topk_ratio=0.01, seed=3)
        g0 = eng.arena.global_w.clone()
        seen = set()
        for _ in range(3):
            eng.run_round(shards, n_epoch=1)
            seen |= set(eng._last_participants)
            k = eng.session.topk_k
            ub = eng.last_upload_bytes()
            assert ub == sparse_upload_bytes(eng.arena.n, eng.session.last_upload_entries(), "bf16")
            assert 0 < eng.session.last_upload_entries() <= 4 * k
        eng.sync()
        torch.cuda.synchronize()
        eng.session.check()
        res = eng.topk_residuals()
        assert set(res) == seen and all(torch.isfinite(e).all() for e in res.values())
        assert k == TopKConfig(0.01).k(n_float(eng.arena))
        return eng.arena.global_w - g0

    a, b, c = run("fused"), run("fused"), run("nccl")
    noise, diff = _rel(b, a), _rel(c, a)
    print("3 top-k rounds, rel diff: fused/fused {:.2e}, fused/nccl {:.2e}".format(noise, diff))
    assert diff <= 3.0 * noise + 2e-2, (diff, noise)


def test_multi_gpu_against_nccl():
    n = torch.cuda.device_count()
    if n < 2:
        pytest.skip("needs 2 or more GPUs")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(min(n, 4)),
           "--master-addr", "127.0.0.1", "--master-port", str(29700 + os.getpid() % 200),
           os.path.join(root, "tests", "mp_topk_check.py")]
    proc = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=600, cwd=root)
    assert proc.returncode == 0 and "RESULT PASS" in proc.stdout, proc.stdout[-4000:]
