"""Personalized federated learning (FedBN / FedPer, parallel/personal.py) on the CPU: the arena layout with a client-local
range, key resolution, the feature rules of the new axis, the NcclSession oracle against a plain session over the
compacted arena, the local store's swaps, and a two-rank gloo run of the engine (tests/mp_personal_gloo.py)."""
import os
import subprocess
import sys

import pytest
import torch
from torch import nn

from baton_b200.models import MLP2, LinearModel, resnet18
from baton_b200.models.bert import bert_tiny
from baton_b200.parallel.arena import ParamArena
from baton_b200.parallel.dp import DPConfig
from baton_b200.parallel.engine import FederatedEngine
from baton_b200.parallel.compress import TopKConfig
from baton_b200.parallel.features import check_features
from baton_b200.parallel.fedavg import NcclSession
from baton_b200.parallel.personal import LocalStore, resolve_local_keys
from baton_b200.parallel.robust import RobustConfig
from baton_b200.parallel.server_opt import ServerOptConfig

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _bn_keys(model):
    from baton_b200.ops.nn import BatchNorm2d
    out = []
    for name, m in model.named_modules():
        if isinstance(m, BatchNorm2d):
            out += [name + "." + leaf for leaf in ("weight", "bias", "running_mean", "running_var")]
    return out


# ---------------------------------------------------------------------------------------------------- layout
@pytest.mark.parametrize("local_keys", ["bn", "head", ("bn", "head")])
def test_resnet_local_range_is_contiguous_aligned_and_straddles_n_param(local_keys):
    torch.manual_seed(0)
    ref = resnet18(10)
    model = resnet18(10)
    model.load_state_dict(ref.state_dict())
    keys = resolve_local_keys(model, local_keys)
    a = ParamArena(model, "cpu", local=keys)
    lo, hi = a.local_range
    assert lo % 1024 == 0 and hi % 1024 == 0 and lo <= a.n_param <= hi and a.n_shared % 1024 == 0
    assert a.n_shared == a.n - (hi - lo)
    for name, s in a.slots.items():
        inside = lo <= s.offset and s.offset + s.numel <= hi
        outside = s.offset + s.numel <= lo or s.offset >= hi
        assert (inside if name in keys else outside), name
        assert s.is_param == (s.offset < a.n_param), name
    # state_dict keys, shapes and values do not see the reorder
    got, want = model.state_dict(), ref.state_dict()
    assert list(got) == list(want)
    for k in want:
        assert got[k].shape == want[k].shape and torch.equal(got[k], want[k]), k


def test_no_local_keys_keeps_todays_offsets():
    torch.manual_seed(0)
    m = resnet18(10)
    a = ParamArena(m, "cpu")
    assert a.local_range is None and a.n_shared == a.n
    off = 0
    for name, p in m.named_parameters():
        assert a.slots[name].offset == off, name
        off = (off + p.numel() + 7) // 8 * 8
    assert a.n_param == off
    for name, b in m.named_buffers():
        if b.is_floating_point():
            assert a.slots[name].offset == off, name
            off = (off + b.numel() + 7) // 8 * 8
    assert a.n == (off + 2047) // 2048 * 2048


def test_fedbn_and_fedper_sizes_on_resnet18():
    m = resnet18(10)
    bn = resolve_local_keys(m, "bn")
    assert sorted(bn) == sorted(_bn_keys(m))
    a = ParamArena(m, "cpu", local=bn)
    lo, hi = a.local_range
    assert sum(a.slots[k].numel for k in bn) == 4 * 4800 and hi - lo == 19456
    m = resnet18(10)
    head = resolve_local_keys(m, "head")
    assert head == ["fc.weight", "fc.bias"]
    a = ParamArena(m, "cpu", local=head)
    assert sum(a.slots[k].numel for k in head) == 5130


# ---------------------------------------------------------------------------------------------------- key resolution
def test_key_resolution_presets_patterns_and_mixes():
    m = resnet18(10)
    assert "bn1.running_mean" in resolve_local_keys(m, "bn")
    assert not any(k.endswith("num_batches_tracked") for k in resolve_local_keys(m, "bn"))
    both = resolve_local_keys(m, ("bn", "head"))
    assert set(both) == set(resolve_local_keys(m, "bn")) | {"fc.weight", "fc.bias"}
    assert resolve_local_keys(m, ["layer1.*.bn?.weight", "fc.bias"]) == \
        [k for k in m.state_dict() if k.startswith("layer1.") and k.endswith(("bn1.weight", "bn2.weight"))] + ["fc.bias"]
    # a pattern over an integer buffer keeps only the float entries
    assert resolve_local_keys(m, "bn1.*") == ["bn1.weight", "bn1.bias", "bn1.running_mean", "bn1.running_var"]
    b = bert_tiny(2)
    assert resolve_local_keys(b, "head") == ["classifier.weight", "classifier.bias"]
    assert resolve_local_keys(MLP2(), "head") == ["fc2.weight", "fc2.bias"]
    assert resolve_local_keys(MLP2(), "fc1.bias") == ["fc1.bias"]


@pytest.mark.parametrize("model, local_keys, match", [
    (MLP2, "bn", "matches no"),                       # no BatchNorm
    (bert_tiny, "bn", "matches no"),
    (resnet18, "nothing.*", "matches no"),
    (resnet18, ("bn", "nothing"), "matches no"),
    (LinearModel, "head", "whole model"),
    (MLP2, ("fc1.*", "head"), "every float"),
    (resnet18, "*", "every float"),
    (resnet18, (), "takes"),
    (resnet18, ("bn", 3), "takes"),
])
def test_key_resolution_errors(model, local_keys, match):
    m = model(10) if model is resnet18 else model()
    with pytest.raises(ValueError, match=match):
        resolve_local_keys(m, local_keys)


def test_head_preset_needs_a_head():
    class NoHead(nn.Module):
        def __init__(self):
            super().__init__()
            self.a = nn.Linear(2, 2)
            self.b = nn.Linear(2, 2)
    with pytest.raises(ValueError, match="head prefix"):
        resolve_local_keys(NoHead(), "head")


# ---------------------------------------------------------------------------------------------------- feature rules
REJECTED = [
    (dict(dp=DPConfig(1.0, 0.5, seed=1)), dict(dp_clip=1.0, dp_noise_multiplier=0.5, dp_seed=1), "DP-FedAvg"),
    (dict(scaffold=True), dict(scaffold=True), "SCAFFOLD"),
    (dict(robust=RobustConfig("median")), dict(aggregator="median"), "robust aggregator"),
    (dict(robust=RobustConfig("krum", krum_f=0)), dict(aggregator="krum"), "robust aggregator or Krum"),
    (dict(topk=TopKConfig(0.1, True)), dict(compress="topk", topk_ratio=0.1), "top-k"),
    (dict(tile_flags=True), dict(tile_flags=True), "tile_flags"),
]


def _reason(fn):
    with pytest.raises(ValueError) as e:
        fn()
    return str(e.value)


@pytest.mark.parametrize("session_kw, engine_kw, word", REJECTED)
def test_every_rule_gives_the_same_reason_at_the_engine_and_the_session(session_kw, engine_kw, word):
    feat = {k: v for k, v in session_kw.items()}
    direct = _reason(lambda: check_features(local=True, **feat))
    assert word in direct and "client-local" in direct
    eng = _reason(lambda: FederatedEngine(MLP2(), "cpu", backend="nccl", loss="mse", local_keys="head",
                                          logical_clients=4, **engine_kw))
    a = ParamArena(MLP2(), "cpu", local=resolve_local_keys(MLP2(), "head"))
    sess = _reason(lambda: NcclSession(a, local=True, max_clients=1, **session_kw))
    assert eng == direct and sess == direct


@pytest.mark.parametrize("session_kw, engine_kw, word", REJECTED)
def test_the_fused_session_gives_the_same_reason(session_kw, engine_kw, word):
    from baton_b200.parallel.fedavg import FedAvgSession
    a = ParamArena(MLP2(), "cpu", local=resolve_local_keys(MLP2(), "head"))
    want = _reason(lambda: check_features(local=True, **session_kw))
    # the rules run before the session touches the device
    got = _reason(lambda: FedAvgSession(a, local=True, **session_kw))
    assert got == want


def test_manager_planes_are_rejected():
    for plane in ("http", "seated"):
        assert "manager plane" in _reason(lambda: check_features(local=True, plane=plane))


@pytest.mark.parametrize("kw", [
    dict(wire_dtype="fp32"), dict(wire_dtype="bf16"), dict(wire_dtype="fp8"), dict(mode="weights"),
    dict(server_opt=ServerOptConfig("adam", 0.1)), dict(prox_mu=0.1), dict(optimizer="adamw"), dict(momentum=0.9),
])
def test_what_combines(kw):
    check_features(local=True, **kw)


def test_session_local_flag_must_match_the_arena():
    plain = ParamArena(MLP2(), "cpu")
    with pytest.raises(ValueError, match="local=True"):
        NcclSession(plain, local=True)
    a = ParamArena(MLP2(), "cpu", local=["fc2.bias"])
    with pytest.raises(ValueError, match="local=True"):
        NcclSession(a)


# ---------------------------------------------------------------------------------------------------- the NCCL oracle
class _Compact(nn.Module):
    """A module whose arena IS the logical vector of a personalized arena: one parameter of lo elements, one buffer of
    n - hi elements."""

    def __init__(self, n_lo, n_tail):
        super().__init__()
        self.p = nn.Parameter(torch.zeros(n_lo))
        self.register_buffer("b", torch.zeros(n_tail))


def _compact_arena(a, momentum):
    lo, hi = a.local_range
    c = ParamArena(_Compact(lo, a.n - hi), "cpu", momentum=momentum, total_align=1024)
    assert c.n == a.n_shared and c.n_param == lo
    return c


def _load(c, a, src):
    lo, hi = a.local_range
    c.theta.copy_(torch.cat((src.theta[:lo], src.theta[hi:])))
    c.global_w.copy_(torch.cat((src.global_w[:lo], src.global_w[hi:])))


@pytest.mark.parametrize("wire_dtype", ["fp32", "bf16"])
@pytest.mark.parametrize("mode, sopt", [("delta", None), ("weights", None), ("delta", "avgm"), ("delta", "adam")])
def test_nccl_session_with_local_equals_a_plain_session_over_the_compacted_arena(wire_dtype, mode, sopt):
    torch.manual_seed(1)
    m = resnet18(10)
    a = ParamArena(m, "cpu", momentum=True, local=resolve_local_keys(m, ("bn", "head")))
    lo, hi = a.local_range
    c = _compact_arena(a, momentum=True)
    g = torch.Generator().manual_seed(5)
    cfg = ServerOptConfig(sopt, 0.1) if sopt else None
    s = NcclSession(a, wire_dtype=wire_dtype, mode=mode, server_opt=cfg, local=True)
    sc = NcclSession(c, wire_dtype=wire_dtype, mode=mode, server_opt=ServerOptConfig(sopt, 0.1) if sopt else None)
    st0 = [t.clone() if t is not None else None for t in s.server_state()] if cfg is not None else []
    for r in range(2):
        a.theta.copy_(a.global_w + 0.01 * torch.randn(a.n, generator=g))
        a.momentum.fill_(3.0)
        before = {k: getattr(a, k).clone() for k in ("theta", "global_w", "theta_bf16", "momentum")}
        _load(c, a, a)
        s.aggregate(my_n=7.0)
        sc.aggregate(my_n=7.0)
        for k in ("theta", "global_w", "theta_bf16"):
            x = getattr(a, k)
            assert torch.equal(torch.cat((x[:lo], x[hi:])), getattr(c, k)), (r, k)
            assert torch.equal(x[lo:hi], before[k][lo:hi]), (r, k)
        assert torch.equal(a.momentum[:lo], torch.zeros(lo)) and torch.equal(a.momentum[lo:], before["momentum"][lo:])
        if cfg is not None:
            for x, y, x0 in zip(s.server_state(), sc.server_state(), st0):
                if x is not None:      # the state over the local parameters keeps its initial values
                    assert torch.equal(x[:lo], y) and torch.equal(x[lo:], x0[lo:])
    assert s.wire_bytes() == sc.wire_bytes() < NcclSession(ParamArena(resnet18(10), "cpu"), wire_dtype=wire_dtype).wire_bytes()


# ---------------------------------------------------------------------------------------------------- the store
def test_store_swaps_are_slice_copies():
    torch.manual_seed(2)
    m = resnet18(10)
    a = ParamArena(m, "cpu", momentum=True, local=resolve_local_keys(m, "bn"))
    lo, hi = a.local_range
    st = LocalStore(a, resolve_local_keys(m, "bn"))
    init = a.theta[lo:hi].clone()
    a.theta.normal_()
    a.global_w.normal_()
    a.momentum.fill_(2.0)
    other = a.theta.clone()
    st.swap_in(3)                                   # first time: the initial values
    assert torch.equal(a.theta[lo:hi], init) and torch.equal(a.global_w[lo:hi], init)
    assert torch.equal(a.theta_bf16[lo:hi], init.to(torch.bfloat16))
    assert not a.momentum[lo: a.n_param].any() and (a.momentum[:lo] == 2.0).all()
    assert torch.equal(a.theta[:lo], other[:lo]) and torch.equal(a.theta[hi:], other[hi:])
    a.theta[lo:hi].add_(1.0)
    st.swap_out(3)
    a.theta[lo:hi].zero_()
    a.momentum.fill_(2.0)
    st.swap_in(3)
    assert torch.equal(a.theta[lo:hi], init + 1.0) and not a.momentum[lo: a.n_param].any()
    e = st.entries(3)
    assert torch.equal(e["bn1.running_var"], m.bn1.running_var) and e["bn1.running_var"].data_ptr() != \
        m.bn1.running_var.data_ptr()
    assert torch.equal(st.initial_entries()["bn1.weight"], init[a.slots["bn1.weight"].offset - lo:][:64])


# ---------------------------------------------------------------------------------------------------- engine on the CPU
def test_engine_api_one_process():
    torch.manual_seed(3)
    eng = FederatedEngine(MLP2(), "cpu", backend="nccl", loss="mse", lr=0.01, batch_size=8, wire_dtype="fp32",
                          logical_clients=3, local_keys="head")
    with pytest.raises(RuntimeError, match="not hosted"):
        eng.client_state_dict(3)
    X = torch.randn(16, 10)
    y = X.sum(1, keepdim=True)
    before = eng.state_dict()
    before = {k: v.clone() for k, v in before.items()}
    eng.run_round(lambda c: (X * (c + 1), y * (c + 1)), n_epoch=1)
    sd = eng.state_dict()
    assert torch.equal(sd["fc2.weight"], before["fc2.weight"])             # local: the initial values
    assert not torch.equal(sd["fc1.weight"], before["fc1.weight"])         # shared: the new global model
    for c in range(3):
        csd = eng.client_state_dict(c)
        assert torch.equal(csd["fc1.weight"], sd["fc1.weight"])
        assert torch.equal(csd["fc2.weight"], eng.local_entries(c)["fc2.weight"])
        assert not torch.equal(csd["fc2.weight"], before["fc2.weight"])
    plain = FederatedEngine(MLP2(), "cpu", backend="nccl", loss="mse")
    with pytest.raises(RuntimeError, match="off"):
        plain.local_entries(0)


def test_two_gloo_ranks_logical_clients_personal_round():
    port = 29400 + ((os.getpid() + 307) % 500)
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2",
           "--master-addr", "127.0.0.1", "--master-port", str(port), os.path.join(ROOT, "tests", "mp_personal_gloo.py")]
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="", OMP_NUM_THREADS="1")
    proc = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=300, cwd=ROOT, env=env)
    tail = "\n".join(proc.stdout.splitlines()[-40:])
    assert proc.returncode == 0 and "RESULT PASS" in proc.stdout, tail
