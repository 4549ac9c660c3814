"""LoRA fine-tuning on the CPU: the adapter semantics against float64, the Hugging-Face state_dict forms, the frozen
range of the arena, the feature rules, local training against plain torch, and a two-rank gloo round
(tests/mp_lora_gloo.py)."""
import copy
import os
import subprocess
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _tiny(**kw):
    from baton_b200.models.bert import LoraConfig, bert_tiny
    return bert_tiny(2, lora=LoraConfig(**kw))


def _ids(n=4, s=16, seed=0):
    g = torch.Generator().manual_seed(seed)
    return torch.randint(0, 1024, (n, s), generator=g)


def _randomise_adapters(m, seed=1):
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for n, p in m.named_parameters():
            if ".lora_" in n:
                p.copy_(torch.randn(p.shape, generator=g) * 0.1)


def test_config_validation():
    from baton_b200.models.bert import LoraConfig
    assert LoraConfig(16, 8).scale == 0.5
    assert LoraConfig(targets=("value", "query")).targets == ("query", "value")
    for bad in (dict(r=4), dict(r=True), dict(alpha=0), dict(alpha=-1.0), dict(targets=()), dict(targets=("qkv",)),
                dict(targets=("query", "query")), dict(freeze_a=1)):
        with pytest.raises(ValueError):
            LoraConfig(**bad)


def test_fresh_lora_model_matches_base_bitwise():
    from baton_b200.models.bert import bert_tiny
    torch.manual_seed(0)
    base = bert_tiny(2)
    m = _tiny(targets=("query", "key", "value", "attn_out", "ffn_in", "ffn_out"))
    m.load_hf_state_dict(base.hf_state_dict())
    assert torch.equal(m(_ids()), base(_ids()))
    train = sorted(n for n, p in m.named_parameters() if p.requires_grad)
    assert all(".lora_" in n or n.startswith("classifier.") for n in train) and "classifier.weight" in train
    assert not any(p.requires_grad for n, p in m.named_parameters() if n.startswith(("pooler.", "embeddings.")))


@pytest.mark.parametrize("targets", [(True, False, True), (True, True, True), (False, True, False)])
def test_linear_adapter_term_against_float64(targets):
    from baton_b200.ops import nn as bnn
    torch.manual_seed(1)
    lin = bnn.Linear(64, 3 * 96)
    lin.add_lora(8, 2.0, targets)
    _randomise_adapters(lin)
    x = torch.randn(5, 64)
    y = lin(x).double()
    xd, w, b = x.double(), lin.weight.double(), lin.bias.double()
    a, bb = lin.lora_A.double(), lin.lora_B.double()
    t = 0
    for i, on in enumerate(targets):
        ref = xd @ w[i * 96:(i + 1) * 96].t() + b[i * 96:(i + 1) * 96]
        if on:
            ref = ref + 2.0 * (xd @ a[t * 8:(t + 1) * 8].t()) @ bb[t * 96:(t + 1) * 96].t()
            t += 1
        assert torch.allclose(y[:, i * 96:(i + 1) * 96], ref, rtol=1e-5, atol=1e-5), i


def test_merged_state_dict_loads_strictly_and_reproduces_logits():
    from baton_b200.models.bert import bert_tiny
    torch.manual_seed(2)
    m = _tiny(targets=("query", "value", "ffn_out"))
    _randomise_adapters(m)
    plain = bert_tiny(2)
    plain.load_hf_state_dict(m.merged_hf_state_dict(), strict=True)
    ids = _ids(seed=3)
    assert torch.allclose(plain(ids), m(ids), rtol=1e-4, atol=1e-5)


def test_lora_state_dict_round_trip_and_size():
    from baton_b200.models.bert import LoraConfig, bert_base
    torch.manual_seed(3)
    m = _tiny()
    _randomise_adapters(m)
    sd = m.lora_state_dict()
    assert "bert.encoder.layer.0.attention.self.query.lora_A.weight" in sd and "classifier.weight" in sd
    assert sd["bert.encoder.layer.1.attention.self.value.lora_B.weight"].shape == (128, 8)
    other = _tiny()
    other.load_lora_state_dict(sd)
    assert all(torch.equal(v, other.lora_state_dict()[k]) for k, v in sd.items())
    with pytest.raises(KeyError):
        other.load_lora_state_dict({k: v for k, v in sd.items() if k != "classifier.bias"})
    big = bert_base(2, lora=LoraConfig(8, 16))
    assert sum(v.numel() for v in big.lora_state_dict().values()) == 296450


def test_arena_frozen_range():
    from baton_b200.models import resnet18
    from baton_b200.models.bert import bert_tiny
    from baton_b200.parallel.arena import ALIGN, ParamArena
    m = _tiny()
    a = ParamArena(m)
    lo, hi = a.frozen_range
    assert lo == a.n_param and lo % 1024 == 0 and hi % 1024 == 0
    assert a.n_shared == a.n - (hi - lo) and a.grad.numel() == a.n_param
    for name, p in m.named_parameters():
        s = a.slots[name]
        assert (lo <= s.offset < hi) == (not p.requires_grad)
        assert (p.grad is None) == (not p.requires_grad)
    # no frozen parameters: parameters packed from 0 at 8-element alignment, as before
    plain = bert_tiny(2)
    b = ParamArena(plain)
    assert b.frozen_range is None and b.n_shared == b.n
    off = 0
    for name, p in plain.named_parameters():
        assert b.slots[name].offset == off
        off = (off + p.numel() + ALIGN - 1) // ALIGN * ALIGN
    assert b.n_param == off
    r = resnet18(10)
    r.fc.weight.requires_grad_(False)
    with pytest.raises(ValueError, match="hand-scheduled"):
        ParamArena(r)


FROZEN_RULES = [(dict(dp_clip=1.0), "DP-FedAvg"), (dict(scaffold=True), "SCAFFOLD"),
                (dict(aggregator="median"), "robust aggregator"), (dict(compress="topk"), "top-k"),
                (dict(secure_agg=True, wire_dtype="fp32"), "secure aggregation"), (dict(tile_flags=True), "tile_flags")]


@pytest.mark.parametrize("opts,what", FROZEN_RULES)
def test_frozen_rules_same_reason_everywhere(opts, what):
    from baton_b200.parallel.engine import FederatedEngine
    from baton_b200.parallel.features import check_features
    from baton_b200.parallel.arena import ParamArena
    from baton_b200.parallel.fedavg import NcclSession
    from baton_b200.parallel.secagg import SecAggConfig
    from baton_b200.parallel.dp import DPConfig
    from baton_b200.parallel.robust import RobustConfig
    from baton_b200.parallel.compress import TopKConfig
    feats = dict(dp=DPConfig(1.0, 0.0, seed=1) if "dp_clip" in opts else None, scaffold=opts.get("scaffold", False),
                 robust=RobustConfig("median", 0.0) if "aggregator" in opts else None,
                 topk=TopKConfig(0.1, True) if "compress" in opts else None,
                 tile_flags=opts.get("tile_flags", False), wire_dtype=opts.get("wire_dtype", "bf16"))
    with pytest.raises(ValueError) as direct:
        check_features(frozen=True, secure_agg=opts.get("secure_agg", False), **feats)
    assert what in str(direct.value)
    with pytest.raises(ValueError) as eng:
        FederatedEngine(_tiny(), "cpu", backend="nccl", **opts)
    assert str(eng.value) == str(direct.value)
    sess = dict(feats, secagg=SecAggConfig() if opts.get("secure_agg") else None)
    with pytest.raises(ValueError) as s:
        NcclSession(ParamArena(_tiny()), **sess)
    assert str(s.value) == str(direct.value)
    with pytest.raises(ValueError, match="frozen parameters with client-local"):
        check_features(frozen=True, local=True)
    with pytest.raises(ValueError, match="SPMD engine"):
        check_features(frozen=True, plane="http")


@pytest.mark.parametrize("optimizer", ["sgd", "adamw"])
def test_cpu_local_training_matches_plain_torch(optimizer):
    from baton_b200.parallel.arena import ParamArena
    from baton_b200.train import PortableLocalSGD
    torch.manual_seed(4)
    m = _tiny(targets=("query", "value", "ffn_in"))
    _randomise_adapters(m)
    ref = copy.deepcopy(m)
    a = ParamArena(m)
    lo, hi = a.frozen_range
    frozen0 = a.theta[lo:hi].clone()
    X, y = _ids(32, 16, seed=5), torch.arange(32) % 2
    kw = dict(lr=0.05, momentum=0.9) if optimizer == "sgd" else dict(lr=1e-3, weight_decay=0.01)
    torch.manual_seed(9)
    PortableLocalSGD(m, a).run(X, y, n_epoch=2, batch_size=8, optimizer=optimizer, **kw)
    assert torch.equal(a.theta[lo:hi], frozen0)
    params = [p for p in ref.parameters() if p.requires_grad]
    opt = torch.optim.SGD(params, **kw) if optimizer == "sgd" else torch.optim.AdamW(params, **kw)
    torch.manual_seed(9)
    perm = torch.randperm(32)
    for _ in range(2):
        for idx in torch.split(perm, 8):
            opt.zero_grad()
            torch.nn.functional.cross_entropy(ref(X[idx]), y[idx]).backward()
            opt.step()
    got, want = m.lora_state_dict(), ref.lora_state_dict()
    for k in want:
        assert torch.allclose(got[k], want[k], rtol=1e-5, atol=1e-7), k


def test_two_gloo_ranks_lora_round():
    port = 29400 + ((os.getpid() + 411) % 500)
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2",
           "--master-addr", "127.0.0.1", "--master-port", str(port), os.path.join(ROOT, "tests", "mp_lora_gloo.py")]
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="", OMP_NUM_THREADS="1")
    proc = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=300, cwd=ROOT, env=env)
    tail = "\n".join(proc.stdout.splitlines()[-40:])
    assert proc.returncode == 0 and "RESULT PASS" in proc.stdout, tail
