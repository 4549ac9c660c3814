"""Top-k uploads with error feedback on the CPU: the host selection rule (parallel/compress.py) against a brute-force
lexsort, the error-feedback identity, topk_combine, the configuration and every exclusion in the engine and both
sessions, compress=None building today's engine, NcclSession rounds against a closed form, and a 2-process gloo run
(``tests/mp_topk_gloo.py``)."""
import math

import numpy as np
import pytest
import torch

from baton_b200.parallel.arena import ParamArena
from baton_b200.parallel.compress import (NAN_KEY, TopKConfig, TopKState, n_float, sparse_upload_bytes, topk_combine,
                                          topk_ef_, topk_keys, topk_select)
from baton_b200.parallel.dp import DPConfig
from baton_b200.parallel.fedavg import NcclSession
from baton_b200.parallel.robust import RobustConfig


def _brute(u, k):
    bits = u.numpy().view(np.uint32).astype(np.int64) & 0x7FFFFFFF
    key = np.where(bits > 0x7F800000, NAN_KEY, bits)
    order = np.lexsort((np.arange(u.numel()), -key))      # key descending, then index ascending
    return np.sort(order[:k])


def _u(kind, n, seed):
    g = torch.Generator().manual_seed(seed)
    u = torch.randn(n, generator=g)
    if kind == "tied":
        u = torch.round(u * 3) / 3
    elif kind == "special":
        u[::7] = float("nan")
        u[1::7] = -float("nan")
        u[3::11] = float("inf")
        u[4::11] = -float("inf")
        u[5::13] = -0.0
        u[6::13] = 0.0
    elif kind == "zero":
        u.zero_()
    return u


@pytest.mark.parametrize("kind", ["random", "tied", "special", "zero"])
@pytest.mark.parametrize("ratio", [1e-9, 0.013, 0.25, 0.5, 1.0])
def test_selection_matches_brute_force(kind, ratio):
    n = 4099
    u = _u(kind, n, seed=7)
    k = TopKConfig(ratio).k(n)
    assert k == max(1, math.ceil(ratio * n))
    assert np.array_equal(topk_select(u, k).numpy(), _brute(u, k))


def test_nan_ranks_above_inf_and_ties_take_lower_index():
    u = torch.tensor([1.0, float("inf"), float("nan"), -2.0, 2.0, -float("nan"), 0.5])
    assert topk_select(u, 1).tolist() == [2]
    assert topk_select(u, 2).tolist() == [2, 5]
    assert topk_select(u, 3).tolist() == [1, 2, 5]
    assert topk_select(u, 4).tolist() == [1, 2, 3, 5]         # |-2| == |2|: the lower index first
    assert int(topk_keys(torch.tensor([-float("nan")]))[0]) == NAN_KEY


@pytest.mark.parametrize("k", [1, 50, 1000])
def test_error_feedback_identity_is_exact(k):
    g = torch.Generator().manual_seed(k)
    theta, glob = torch.randn(1000, generator=g), torch.randn(1000, generator=g)
    e = torch.randn(1000, generator=g) * 1e-3
    u = (theta - glob) + e
    idx, vals = topk_ef_(theta, glob, e, k)
    top = torch.zeros(1000)
    top[idx] = vals
    assert torch.equal((top + e).view(torch.int32), u.view(torch.int32))
    assert int((e[idx] != 0).sum()) == 0 and idx.numel() == k
    idx2, vals2 = topk_ef_(theta, glob, None, k)                # without error feedback: u = theta - global
    assert torch.equal(idx2, topk_select(theta - glob, k))


def test_topk_combine_is_the_fused_reduce():
    g = torch.Generator().manual_seed(3)
    n = 2048
    lists = []
    for r in range(3):
        idx = torch.sort(torch.randperm(n, generator=g)[:300]).values
        lists.append((idx, torch.randn(300, generator=g)))
    w = [0.25, 0.0, 0.75]
    got = topk_combine(lists + [None], w + [0.5], n, "fp32")
    want = torch.zeros(n)
    for (idx, v), wr in zip(lists, w):
        if wr:
            want[idx] = (v.double() * wr + want[idx].double()).float()
    assert torch.equal(got, want)
    one = topk_combine([lists[0]], [1.0], n, "bf16")
    dense = torch.zeros(n)
    dense[lists[0][0]] = lists[0][1]
    assert torch.equal(one, dense.to(torch.bfloat16).float())


@pytest.mark.parametrize("bad", [0, 0.0, -0.1, 1.5, float("nan"), float("inf"), True, "0.1"])
def test_config_validation(bad):
    with pytest.raises(ValueError):
        TopKConfig(bad)


def test_state_allocates_zero_residuals_once():
    st = TopKState(16, "cpu")
    e = st.residual(3)
    e.add_(1.0)
    assert st.residual(3) is e and set(st.e) == {3} and torch.equal(st.residual(5), torch.zeros(16))


class _Net(torch.nn.Module):
    def __init__(self):
        super().__init__()
        self.fc = torch.nn.Linear(30, 40)
        self.bn = torch.nn.BatchNorm1d(40)

    def forward(self, x):
        return self.bn(self.fc(x))


def _arena():
    torch.manual_seed(0)
    return ParamArena(_Net(), torch.device("cpu"))


def test_n_float_counts_state_dict_floats_without_padding():
    a = _arena()
    floats = sum(v.numel() for v in _Net().state_dict().values() if v.is_floating_point())
    assert n_float(a) == floats < a.n


EXCLUDED = {
    "fp8": dict(wire_dtype="fp8"),
    "dp": dict(dp=DPConfig(1.0, 0.5, seed=1)),
    "robust": dict(robust=RobustConfig("median")),
    "scaffold": dict(scaffold=True),
    "weights": dict(mode="weights"),
    "tile_flags": dict(tile_flags=True),
}


@pytest.mark.parametrize("case", list(EXCLUDED))
def test_sessions_reject_the_exclusions(case):
    from baton_b200.parallel.fedavg import FedAvgSession
    for Session in (NcclSession, FedAvgSession):
        with pytest.raises(ValueError):
            Session(_arena(), topk=TopKConfig(0.1), **EXCLUDED[case])
    with pytest.raises(TypeError):
        NcclSession(_arena(), topk=0.1)


ENGINE_EXCLUDED = {
    "fp8": dict(wire_dtype="fp8"),
    "dp": dict(dp_clip=1.0, dp_noise_multiplier=0.5),
    "median": dict(aggregator="median"),
    "krum": dict(aggregator="krum"),
    "scaffold": dict(scaffold=True),
    "weights": dict(mode="weights"),
    "tile_flags": dict(tile_flags=True),
    "ratio": dict(topk_ratio=0.0),
}


@pytest.mark.parametrize("case", list(ENGINE_EXCLUDED))
def test_engine_rejects_the_exclusions(case):
    from baton_b200.parallel.engine import FederatedEngine
    with pytest.raises(ValueError):
        FederatedEngine(_Net(), "cpu", backend="nccl", compress="topk", **ENGINE_EXCLUDED[case])


def test_engine_compress_none_builds_todays_engine():
    from baton_b200.parallel.engine import FederatedEngine
    with pytest.raises(ValueError):
        FederatedEngine(_Net(), "cpu", backend="nccl", compress="lz4")
    eng = FederatedEngine(_Net(), "cpu", backend="nccl")
    assert eng.topk is None and eng.topk_state is None and eng.session.topk is None
    assert eng.session.max_clients == 1 and eng.last_upload_bytes() == eng.session.wire_bytes()
    with pytest.raises(RuntimeError):
        eng.topk_residuals()
    eng2 = FederatedEngine(_Net(), "cpu", backend="nccl", logical_clients=4, sample_k=3)
    assert eng2.session.topk is None and eng2.session.max_clients == 1
    t = FederatedEngine(_Net(), "cpu", backend="nccl", compress="topk", topk_ratio=0.1, logical_clients=4, sample_k=3)
    assert t.session.topk == TopKConfig(0.1) and t.session.max_clients == 3 and t.topk_residuals() == {}


def test_nccl_session_rounds_match_the_closed_form():
    """Three single-rank rounds with error feedback: global += cast(topk(delta + e)), e carries the rest."""
    a = _arena()
    s = NcclSession(a, wire_dtype="fp32", topk=TopKConfig(0.05))
    k = s.topk_k
    e = torch.zeros(a.n)
    x, e_ref = a.global_w.clone(), torch.zeros(a.n)
    g = torch.Generator().manual_seed(5)
    for r in range(3):
        d = torch.randn(a.n, generator=g) * 0.01
        a.theta.copy_(a.global_w + d)
        u = (a.theta - a.global_w) + e_ref
        idx = torch.from_numpy(_brute(u, k))
        top = torch.zeros(a.n)
        top[idx] = u[idx]
        e_ref = u - top
        x = x + top
        s.pack_topk(e)
        s.aggregate(my_n=4.0)
        assert torch.equal(a.global_w, x) and torch.equal(e, e_ref)
        assert s.last_upload_entries() == k
        assert s.last_upload_bytes() == sparse_upload_bytes(a.n, k, "fp32")


def test_ratio_one_nccl_session_is_the_plain_session():
    a, b = _arena(), _arena()
    sa, sb = NcclSession(a, wire_dtype="bf16", topk=TopKConfig(1.0)), NcclSession(b, wire_dtype="bf16")
    e = torch.zeros(a.n)
    g = torch.Generator().manual_seed(9)
    for r in range(3):
        d = torch.randn(a.n, generator=g) * 0.01
        for arena in (a, b):
            for sl in arena.slots.values():
                arena.theta[sl.offset: sl.offset + sl.numel] += d[sl.offset: sl.offset + sl.numel]
        sa.pack_topk(e)
        sa.aggregate(my_n=2.0)
        sb.aggregate(my_n=2.0)
        assert torch.equal(a.global_w, b.global_w) and int(torch.count_nonzero(e)) == 0


def test_topk_rounds_on_gloo_match_a_host_replay():
    import os
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    port = 29400 + ((os.getpid() + 1777) % 500)
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2",
           "--master-addr", "127.0.0.1", "--master-port", str(port), os.path.join(root, "tests", "mp_topk_gloo.py")]
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="", OMP_NUM_THREADS="1")
    proc = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=300, cwd=root,
                          env=env)
    tail = "\n".join(proc.stdout.splitlines()[-40:])
    assert proc.returncode == 0 and "RESULT PASS" in proc.stdout, tail
